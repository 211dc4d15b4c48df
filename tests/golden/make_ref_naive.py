"""Regenerate tests/golden/ref_naive.npz: the outputs of the reference's own Naive<> (include/Utility.h:18-42,
compiled by oracle/build.py into oracle/_ref/, which needs a reference checkout) on the inputs of
tests/test_oracle.py's REF_CASES, with the oracle's fill recipe (seed 7) and with the special-value inputs
(seed 11).  The tests compare the oracle restatement with these arrays bit for bit.

    python tests/golden/make_ref_naive.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
import oracle as O  # noqa: E402
from oracle import build as oracle_build  # noqa: E402
import test_oracle as T  # noqa: E402


def main():
    oracle_build.build_oracle()
    oracle_build.build_ref(sim=False)
    out = {}
    for dt, mp, rd, ta, (n, k, m) in T.REF_CASES:
        dtype, m_, r_ = getattr(O, dt), getattr(O, mp), getattr(O, rd)
        assert O.ref_available(dtype, m_, r_, ta), (dt, mp, rd, ta)
        a, b = O.fill(dtype, n, k, m, seed=7)
        out[T.ref_key(dt, mp, rd, ta, "fill")] = O.ref_naive(dtype, m_, r_, a, b, n, k, m, transposed_a=ta)
        if dt in T.SPECIAL_DTYPES:
            a, b = T._special_inputs(T.SPECIAL_DTYPES[dt], n, k, m, seed=11)
            out[T.ref_key(dt, mp, rd, ta, "special")] = O.ref_naive(dtype, m_, r_, a, b, n, k, m, transposed_a=ta)
    np.savez_compressed(os.path.join(HERE, "ref_naive.npz"), **out)


if __name__ == "__main__":
    main()
