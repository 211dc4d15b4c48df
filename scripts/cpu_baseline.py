#!/usr/bin/env python
"""CPU baseline of the reference's own path, timed on THIS host's cores (run it on the GPU machine):
  * the reference's Naive<> (include/Utility.h:18-42, compiled in place into oracle/_ref), single
    thread as written, at 256^3 / 1024^3 / 2048^3 (sampled rows at 2048^3) per configuration;
  * the reference's full TestSimulation (thread-per-stage software simulation of the FPGA kernel,
    built from its unmodified sources against oracle/shim) at 256^3 where the binary exists.
Output: JSON (BASELINE.md section 2's table).  Test infrastructure; the product is not involved."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import oracle as O  # noqa: E402

out = {"host_cpus": os.cpu_count(), "cpu_model": "", "naive": [], "test_simulation": []}
try:
    out["cpu_model"] = [l.split(":", 1)[1].strip() for l in open("/proc/cpuinfo") if l.startswith("model name")][0]
except Exception:
    pass
CFGS = [(O.FLOAT, O.MULTIPLY, O.ADD), (O.DOUBLE, O.MULTIPLY, O.ADD), (O.HALF, O.MULTIPLY, O.ADD),
        (O.FLOAT, O.ADD, O.MIN), (O.INT32, O.MULTIPLY, O.ADD)]
for dt, mp, rd in CFGS:
    if not O.ref_available(dt, mp, rd):
        continue
    for size, rows in ((256, 256), (1024, 1024), (2048, 64)):
        if dt == O.HALF and size > 256:
            continue  # the shim's per-operation binary16 emulation is 30x slower; 256^3 is enough
        a, b = O.fill(dt, size, size, size)
        t0 = time.perf_counter()
        O.ref_naive(dt, mp, rd, a[: rows * size], b, rows, size, size)
        dt_s = time.perf_counter() - t0
        out["naive"].append({"config": O.ref_config_name(dt, mp, rd), "shape": [size, size, size],
                             "rows_computed": rows, "seconds": dt_s, "gops": 2e-9 * rows * size * size / dt_s,
                             "threads": 1})
        print(out["naive"][-1], flush=True)
for cfg in ("float_Multiply_Add", "double_Multiply_Add", "int_Multiply_Add"):
    exe = os.path.join(ROOT, "oracle", "_ref", "TestSimulation_" + cfg)
    if os.path.exists(exe):
        t0 = time.perf_counter()
        r = subprocess.run([exe, "256", "256", "256"], capture_output=True, text=True)
        out["test_simulation"].append({"config": cfg, "shape": [256, 256, 256], "seconds": time.perf_counter() - t0,
                                       "verified": "successfully verified" in r.stdout, "rc": r.returncode})
        print(out["test_simulation"][-1], flush=True)
print(json.dumps(out))
