"""The witness suite without a GPU: tests/witness_naive.py is the definition it claims to be, the data of
tests/witness_data.py rejects plausible wrong witness implementations, and the machine code of every
semiring_witness_*.o keeps to its register and arithmetic budget.

* witness_naive's C equals the oracle's Naive<> (tests/bf16_naive.py for bfloat16) bit for bit on the coverage data
  of every (type, Map, Min | Max).  On the FMNMX path (float without MM_FLAG_EXACT) the comparison leaves out the
  elements with a NaN term, where fminf / fmaxf and the literal Min / Max differ by definition.
* witness_naive equals a plain scalar Python loop at tiny shapes, on both paths.
* Mutants: each defect changes W on the data of every pair, except where named in SURVIVES.
* SASS: no local memory (LDL / STL), no FMA contraction in the floating types, UTMALDG in the ring kernel, FMNMX in
  the float default kernels.
"""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import semiring_data as sd  # noqa: E402
import witness_data as wd  # noqa: E402
import witness_naive as wn  # noqa: E402
from semiring_data import AND, FLOAT, FLOATING, MAX, MIN  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "gemm_hls_b200", "build")
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
SEED = 5

# (type, Map, reduce, FMNMX path)
CASES = [(dt, mp, rd, False) for dt in sd.TYPES for mp in sd.OPS for rd in (MIN, MAX)] + \
        [(FLOAT, mp, rd, True) for mp in sd.OPS for rd in (MIN, MAX)]


def _id(c):
    return sd.pair_name(*c[:3]) + ("-fmnmx" if c[3] else "")


_REF = {}


def ref(dt, mp, rd, fm):
    key = (dt, mp, rd, fm)
    if key not in _REF:
        n, m, k = sd.gpu_shape(dt)
        a, b = wd.case(dt, mp, rd, n, k, m, SEED)
        _REF[key] = (a, b) + wn.witness(dt, mp, rd, a, b, fmnmx=fm)
    return _REF[key]


def _has_nan_term(dt, mp, a, b):
    """Elements with a NaN term under the literal Maps (B carries the NaNs of the data)."""
    if dt not in FLOATING or mp == AND:
        return np.zeros((a.shape[0], b.shape[1]), bool)
    nb = sd._Arith(dt).load(b)
    return np.broadcast_to(np.isnan(nb).any(axis=0)[None, :], (a.shape[0], b.shape[1]))


@pytest.mark.parametrize("case", CASES, ids=[_id(c) for c in CASES])
def test_c_is_naive(oracle, case):
    dt, mp, rd, fm = case
    n, m, k = sd.gpu_shape(dt)
    a, b, c, _ = ref(dt, mp, rd, fm)
    want = sd.reference(oracle, dt, mp, rd, a, b, n, k, m)
    if not fm:
        assert sd.same(c, want)
    else:   # fminf / fmaxf drop NaN terms; elsewhere (no -0 in the data) they are the literal Min / Max
        keep = ~_has_nan_term(dt, mp, a, b)
        assert keep.sum() > c.size // 2
        assert sd.same(c[keep], want[keep])


@pytest.mark.parametrize("case", CASES, ids=[_id(c) for c in CASES])
def test_equals_scalar_loop(case):
    dt, mp, rd, fm = case
    n, m, k = 5, 6, 2 * sd.bk(dt)
    a, b = wd.case(dt, mp, rd, 259, k, 210, SEED)
    rows = [0, 3, 130, 258, 7]                      # a k-tile window, k = 0 / K - 1 windows, ROW_ID, ROW_NONE
    cols = [0, 3, 131, 200, 14, 5]                  # a column window, NaN, COL_ID, COL_NONE
    a, b = np.ascontiguousarray(a[rows]), np.ascontiguousarray(b[:, cols])
    c1, w1 = wn.witness(dt, mp, rd, a, b, fmnmx=fm)
    c2, w2 = wn.scalar(dt, mp, rd, a, b, fmnmx=fm)
    assert sd.same(c1, c2) and np.array_equal(w1, w2)
    assert c1.shape == (n, m)


def test_the_data_has_what_the_witness_needs():
    """Winners in every k-tile, at k = 0 and k = K - 1 and at both positions of a pair; ties that decide W; NONE
    where the identity is never beaten."""
    for dt, mp, rd, fm in CASES:
        _, _, k = sd.gpu_shape(dt)
        a, b, c, w = ref(dt, mp, rd, fm)
        hit = w[w != wn.NONE]
        name = _id((dt, mp, rd, fm))
        assert set((hit // sd.bk(dt)).tolist()) == set(range(k // sd.bk(dt))), name
        assert (hit == 0).any() and (hit == k - 1).any(), name
        assert (hit % 2 == 0).any() and (hit % 2 == 1).any(), name
        _, w_tie = wn.witness(dt, mp, rd, a, b, fmnmx=fm, tie="swapped")
        assert (w_tie != w).sum() > 100, name
        ident = w[wd.ROW_ID, wd.COL_ID]
        if mp != AND:
            assert ident == (wn.NONE if fm else k - 1), name
        if dt in FLOATING and mp != AND:
            assert (w[wd.ROW_NONE] == wn.NONE).any(), name
        if dt in FLOATING and mp != AND and not fm:
            assert np.isnan(sd._Arith(dt).load(b)).any(), name


# Mutant -> pairs on whose data it cannot show (and why).  NONE only exists where a term can be worse than the
# identity: never for integers (every term ties or beats numeric_limits max / min), and never for And under Min
# (its terms 0 and 1 are below numeric_limits::max()).
def _no_none(dt, mp, rd, fm):
    return dt not in FLOATING or (mp == AND and rd == MIN)


SURVIVES = {"none_as_0": _no_none, "none_as_K": _no_none}
MUTANTS = {
    "tie_swapped": lambda k, fm: dict(tie="swapped"),
    "pair_order_swapped": lambda k, fm: dict(pair_order="swapped"),
    "off_by_one": lambda k, fm: dict(offset=1),
    "off_by_minus_one": lambda k, fm: dict(offset=-1),
    "none_as_0": lambda k, fm: dict(none=0),
    "none_as_K": lambda k, fm: dict(none=k),
    "other_path_rule": lambda k, fm: dict(rule="literal" if fm else "fmnmx"),
    "once_per_k_tile": lambda k, fm: dict(per_tile=True),
}


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_the_data_rejects_the_mutant(mutant):
    shown, hidden = [], []
    for dt, mp, rd, fm in CASES:
        _, _, k = sd.gpu_shape(dt)
        a, b, _, w = ref(dt, mp, rd, fm)
        _, wm = wn.witness(dt, mp, rd, a, b, fmnmx=fm, **MUTANTS[mutant](k, fm))
        (hidden if np.array_equal(wm, w) else shown).append((dt, mp, rd, fm))
    expected_hidden = [c for c in CASES if SURVIVES.get(mutant, lambda *x: False)(*c)]
    assert hidden == expected_hidden, [_id(c) for c in hidden]
    assert shown


def test_k_counted_over_the_batch_shows_from_the_second_problem():
    """W = k + z K (k counted over a batch) equals W on problem 0 and can only show from problem 1 on: there every
    W != NONE moves out of [0, K)."""
    dt, mp, rd = FLOAT, sd.ADD, MIN
    _, _, k = sd.gpu_shape(dt)
    a, b, _, w = ref(dt, mp, rd, False)
    _, w1 = wn.witness(dt, mp, rd, a, b, k_origin=k)
    assert (w1 != w).sum() == (w != wn.NONE).sum() > 0


# ---- machine code ----------------------------------------------------------------------------------------------

def _functions(obj):
    path = os.path.join(OBJ, obj)
    if not os.path.exists(path):
        from gemm_hls_b200 import build as product_build
        product_build.build(force=True)   # the library may be current while its objects were left behind
    text = subprocess.run([CUOBJDUMP, "-sass", path], capture_output=True, text=True, check=True).stdout
    funcs, name = {}, None
    for line in text.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs[name] = []
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][^;]*);", line)   # addresses past 0xffff too
        if m and name:
            funcs[name].append(m.group(1).strip())
    return funcs


def _count(ops, prefix):
    return sum(1 for o in ops if o.startswith(prefix))


def _register_sources(instruction):
    operands = [o.strip() for o in instruction.split(None, 1)[1].split(",")][1:]
    return sum(1 for o in operands if re.match(r"^[-|~]*R\d+", o))


OBJECTS = [("semiring_witness_%s_%d.o" % (s, mp), s) for s in ("f16", "f32", "f64", "i32", "u32", "u8", "bf16")
           for mp in range(7 if s == "f32" else 5)]


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not installed")
@pytest.mark.parametrize("obj,suffix", OBJECTS, ids=[o for o, _ in OBJECTS])
def test_witness_sass(mm, obj, suffix):
    funcs = {n: ops for n, ops in _functions(obj).items() if "semiring_witness_" in n}
    four = suffix in ("f32", "i32", "u32")
    reduces = 4 if suffix == "f32" else 2
    assert len(funcs) == reduces * (2 if four else 1), sorted(funcs)
    for name, ops in funcs.items():
        assert _count(ops, "LDL") == 0 and _count(ops, "STL") == 0, name            # no spills
        bad = [o for o in ops if o.startswith(("FFMA", "DFMA", "HFMA")) and _register_sources(o) >= 3]
        assert not bad, (name, bad[:4])                                            # no contracted Map-Reduce
        if "ring_kernel" in name:
            assert _count(ops, "UTMALDG") >= 2 and _count(ops, "BAR") <= 2, name   # both tiles by TMA
        if "7MinFast" in name or "7MaxFast" in name:
            assert _count(ops, "FMNMX") >= (1024 if "ring_kernel" in name else 64), name   # C stays FMNMX
