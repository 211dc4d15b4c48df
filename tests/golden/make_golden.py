#!/usr/bin/env python
"""Generate tests/golden/golden.json from the REFERENCE'S OWN Naive<> (include/Utility.h:18-42).

Needs a reference checkout ($MM_REFERENCE_DIR) to build oracle/_ref:
    python oracle/build.py && python tests/golden/make_golden.py
Every record is produced by oracle/_ref/libref_naive_<cfg>.so — the reference's template compiled
in place — on inputs drawn with the reference's recipe (seed 5, U[1,10], A then B;
test/TestSimulation.cpp:42-55).  The committed JSON is what the tests read.
"""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import oracle as O  # noqa: E402

CASES = [
    # (dtype, map, reduce, transposed_a, [(n, k, m), ...])
    (O.FLOAT, O.MULTIPLY, O.ADD, False, [(256, 256, 256), (513, 528, 528), (1024, 1024, 1024)]),
    (O.DOUBLE, O.MULTIPLY, O.ADD, False, [(256, 256, 256), (513, 528, 528)]),
    (O.INT32, O.MULTIPLY, O.ADD, False, [(256, 256, 256), (513, 528, 528)]),
    (O.UINT32, O.MULTIPLY, O.ADD, False, [(256, 256, 256)]),
    (O.UINT8, O.MULTIPLY, O.ADD, False, [(256, 256, 256), (130, 192, 128)]),
    (O.FLOAT, O.ADD, O.MIN, False, [(256, 256, 256), (513, 528, 528)]),
    (O.FLOAT, O.ADD, O.MAX, False, [(256, 256, 256)]),
    (O.FLOAT, O.MIN, O.MAX, False, [(256, 256, 256)]),
    (O.DOUBLE, O.ADD, O.MIN, False, [(256, 256, 256)]),
    (O.INT32, O.ADD, O.MIN, False, [(256, 256, 256)]),
    (O.INT32, O.AND, O.ADD, False, [(256, 256, 256)]),
    (O.HALF, O.MULTIPLY, O.ADD, False, [(128, 64, 128)]),
    (O.FLOAT, O.MULTIPLY, O.ADD, True, [(256, 256, 256), (129, 144, 160)]),
]


def record(dtype, mp, rd, ta, n, k, m):
    a, b = O.fill(dtype, n, k, m)
    c = O.ref_naive(dtype, mp, rd, a, b, n, k, m, transposed_a=ta)
    c64 = c.astype(np.float64)
    return {
        "config": O.ref_config_name(dtype, mp, rd, ta),
        "dtype": dtype, "map": mp, "reduce": rd, "transposed_a": ta,
        "n": n, "k": k, "m": m, "seed": 5,
        "a0": repr(float(a[0])), "a1": repr(float(a[1])), "b0": repr(float(b[0])),
        "a_sha256": hashlib.sha256(a.tobytes()).hexdigest(),
        "b_sha256": hashlib.sha256(b.tobytes()).hexdigest(),
        "c_first": repr(float(c64.flat[0])), "c_last": repr(float(c64.flat[-1])),
        "c_sum": repr(float(c64.sum())),
        "c_sha256": hashlib.sha256(c.tobytes()).hexdigest(),
        "source": "reference Naive<> (include/Utility.h:18-42) via oracle/_ref, g++ -O2 -std=c++14",
    }


def main():
    out = []
    for dtype, mp, rd, ta, shapes in CASES:
        for (n, k, m) in shapes:
            r = record(dtype, mp, rd, ta, n, k, m)
            print(r["config"], n, k, m, r["c_first"], r["c_last"], r["c_sum"])
            out.append(r)
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
