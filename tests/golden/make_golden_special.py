#!/usr/bin/env python
"""Generate tests/golden/golden_special.json from the REFERENCE'S OWN Naive<> (include/Utility.h:18-42) on inputs the
reference's recipe never produces: mixed signs, NaN / -0 / +0 / infinities, full-range bytes
(tests/golden/special_inputs.py).  Needs a reference checkout ($MM_REFERENCE_DIR) for oracle/_ref:
    python oracle/build.py && python tests/golden/make_golden_special.py
"""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
import oracle as O  # noqa: E402
import special_inputs as S  # noqa: E402

CASES = [
    # (dtype, map, reduce, input kind, seed, (n, k, m))
    (O.UINT8, O.MULTIPLY, O.ADD, "bytes", 41, (513, 576, 576)),      # 8-bit tensor cores: the modulo-256 wrap-around
    (O.UINT8, O.MULTIPLY, O.ADD, "bytes", 42, (129, 128, 192)),
    (O.FLOAT, O.ADD, O.MIN, "signed", 51, (257, 192, 144)),          # default flags (FMNMX) territory: no NaN, no zeros
    (O.FLOAT, O.ADD, O.MAX, "signed", 52, (65, 32, 48)),
    (O.FLOAT, O.MIN, O.MAX, "signed", 53, (65, 32, 48)),
    (O.INT32, O.ADD, O.MIN, "signed", 54, (130, 64, 96)),
    (O.INT32, O.MULTIPLY, O.ADD, "signed", 55, (130, 64, 96)),
    (O.FLOAT, O.ADD, O.MIN, "special", 61, (65, 32, 48)),            # MM_FLAG_EXACT territory
    (O.FLOAT, O.ADD, O.MAX, "special", 62, (65, 32, 48)),
    (O.FLOAT, O.MIN, O.MAX, "special", 63, (65, 32, 48)),
    (O.FLOAT, O.MULTIPLY, O.ADD, "special", 64, (65, 32, 48)),
    (O.DOUBLE, O.MULTIPLY, O.ADD, "special", 65, (65, 16, 24)),
    (O.DOUBLE, O.ADD, O.MIN, "special", 66, (65, 16, 24)),
    (O.HALF, O.MULTIPLY, O.ADD, "special", 67, (65, 64, 96)),
]


def main():
    out = []
    for dtype, mp, rd, kind, seed, (n, k, m) in CASES:
        assert O.ref_available(dtype, mp, rd), O.ref_config_name(dtype, mp, rd)
        a, b = S.make(kind, O.NP_DTYPE[dtype], n, k, m, seed)
        c = O.ref_naive(dtype, mp, rd, a, b, n, k, m)
        out.append({
            "config": O.ref_config_name(dtype, mp, rd), "dtype": dtype, "map": mp, "reduce": rd, "inputs": kind,
            "seed": seed, "n": n, "k": k, "m": m,
            "a_sha256": hashlib.sha256(a.tobytes()).hexdigest(), "b_sha256": hashlib.sha256(b.tobytes()).hexdigest(),
            "c_sha256_nan_canonical": S.canonical_sha256(c),
            "c_nan_count": int(np.isnan(c.astype(np.float64)).sum()) if np.issubdtype(c.dtype, np.floating) else 0,
            "source": "reference Naive<> (include/Utility.h:18-42) via oracle/_ref, g++ -O2 -std=c++14",
        })
        print(out[-1]["config"], kind, n, k, m, "NaNs in C:", out[-1]["c_nan_count"])
    with open(os.path.join(HERE, "golden_special.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
