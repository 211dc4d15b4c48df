#!/usr/bin/env python
"""Build recipe for the oracle (TEST INFRASTRUCTURE, never shipped in the product).

  python oracle/build.py            # oracle restatement + (if a reference checkout exists) oracle/_ref
  python oracle/build.py --ref-sim  # additionally the reference's full TestSimulation binaries

Outputs
  oracle/liboracle.so                       my restatement (oracle/naive.cpp)
  oracle/_ref/libref_naive_<cfg>.so         the reference's own Naive<> (include/Utility.h:18-42),
                                            compiled in place from $MM_REFERENCE_DIR
  oracle/_ref/TestSimulation_<cfg>          the reference's kernel simulation + test main
                                            (kernel/{Compute,Memory,Top}.cpp, test/TestSimulation.cpp)
  oracle/_ref/cfg_<cfg>/Config.h            what CMake's configure_file(include/Config.h.in) would emit
                                            (CMakeLists.txt:136) for that configuration

No reference source is copied into the repository: the compiler reads the files where they
lie; only generated Config.h and binaries land in oracle/_ref/ (git-ignored).
The reference's own build system (CMake + FindVitis) is NOT run: it requires Vitis.
"""
import argparse
import os
import re
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("MM_REFERENCE_DIR", "/root/reference")
OUT = os.path.join(HERE, "_ref")

# CMake cache defaults, CMakeLists.txt:16-36
DEFAULTS = dict(
    MM_DATA_TYPE="float", MM_MEMORY_BUS_WIDTH_N=64, MM_MEMORY_BUS_WIDTH_K=64,
    MM_MEMORY_BUS_WIDTH_M=64, MM_SIZE_N=512, MM_SIZE_K=512, MM_SIZE_M=512,
    MM_MEMORY_TILE_SIZE_N=256, MM_MEMORY_TILE_SIZE_M=256, MM_PARALLELISM_N=32,
    MM_PARALLELISM_M=8, MM_TRANSPOSE_WIDTH=64, MM_MAP_OP="Multiply", MM_REDUCE_OP="Add",
    MM_CLOCK_INTERNAL=300, MM_GOLDEN_DIR="", MM_TRANSPOSED_A=False)
WIDTH = {"float": 4, "double": 8, "half": 2, "int": 4, "unsigned": 4, "unsigned int": 4,
         "uint8_t": 1, "char": 1, "short": 2, "long": 8}

# (name, overrides).  MM_PARALLELISM_M must divide the bus width in elements (CMakeLists.txt:60-63).
REF_CONFIGS = [
    ("float_Multiply_Add", {}),
    ("double_Multiply_Add", dict(MM_DATA_TYPE="double", MM_PARALLELISM_M=4)),
    ("int_Multiply_Add", dict(MM_DATA_TYPE="int")),
    ("unsigned_Multiply_Add", dict(MM_DATA_TYPE="unsigned")),
    ("uint8_t_Multiply_Add", dict(MM_DATA_TYPE="uint8_t")),
    ("float_Add_Min", dict(MM_MAP_OP="Add", MM_REDUCE_OP="Min")),
    ("float_Add_Max", dict(MM_MAP_OP="Add", MM_REDUCE_OP="Max")),
    ("float_Min_Max", dict(MM_MAP_OP="Min", MM_REDUCE_OP="Max")),
    ("double_Add_Min", dict(MM_DATA_TYPE="double", MM_PARALLELISM_M=4, MM_MAP_OP="Add", MM_REDUCE_OP="Min")),
    ("int_Add_Min", dict(MM_DATA_TYPE="int", MM_MAP_OP="Add", MM_REDUCE_OP="Min")),
    ("int_And_Add", dict(MM_DATA_TYPE="int", MM_MAP_OP="And", MM_REDUCE_OP="Add")),
    ("half_Multiply_Add", dict(MM_DATA_TYPE="half", MM_PARALLELISM_M=16)),
    ("float_Multiply_Add_TA", dict(MM_TRANSPOSED_A=True)),
]
# Configurations for which the reference's full simulation is also built.
SIM_CONFIGS = ["float_Multiply_Add", "double_Multiply_Add", "int_Multiply_Add"]


def run(cmd):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        raise RuntimeError("command failed: " + cmd[0])
    return r


def build_oracle():
    out = os.path.join(HERE, "liboracle.so")
    src = os.path.join(HERE, "naive.cpp")
    if os.path.exists(out) and os.path.getmtime(out) >= os.path.getmtime(src):
        return out
    run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-pthread", "-o", out, src])
    return out


def emit_config(name, overrides):
    cfg = dict(DEFAULTS)
    cfg.update(overrides)
    dt = cfg["MM_DATA_TYPE"]
    cfg["MM_DATA_WIDTH_" + dt] = WIDTH[dt]
    cfg["MM_KERNEL_WIDTH_M"] = WIDTH[dt] * cfg["MM_PARALLELISM_M"]   # CMakeLists.txt:52
    cfg["MM_KERNEL_WIDTH_N"] = WIDTH[dt] * cfg["MM_PARALLELISM_N"]   # CMakeLists.txt:51
    text = open(os.path.join(REF, "include", "Config.h.in")).read()
    for _ in range(2):  # ${MM_DATA_WIDTH_${MM_DATA_TYPE}} nests one level
        text = re.sub(r"\$\{([A-Za-z0-9_ ]+)\}", lambda mo: str(cfg.get(mo.group(1), "")), text)
    d = os.path.join(OUT, "cfg_" + name)
    os.makedirs(d, exist_ok=True)
    path = os.path.join(d, "Config.h")
    if not (os.path.exists(path) and open(path).read() == text):
        open(path, "w").write(text)
    return d, cfg


def common_flags(cfg_dir, cfg):
    flags = ["-std=c++14", "-O2", "-pthread", "-w", "-DMM_DYNAMIC_SIZES",
             "-DHLSLIB_STREAM_TIMEOUT=16", "-DHLSLIB_LEGACY_SDX=0",   # CMakeLists.txt:98-109
             "-I" + cfg_dir, "-I" + os.path.join(HERE, "shim"),
             "-I" + os.path.join(REF, "include"), "-I" + os.path.join(REF, "hlslib", "include")]
    if cfg["MM_TRANSPOSED_A"]:
        flags.append("-DMM_TRANSPOSED_A")
    if cfg["MM_DATA_TYPE"] == "half":
        flags.append("-DMM_HALF_PRECISION")
    return flags


def build_ref_naive(name, overrides):
    cfg_dir, cfg = emit_config(name, overrides)
    out = os.path.join(OUT, "libref_naive_%s.so" % name)
    if os.path.exists(out):
        return out
    run(["g++"] + common_flags(cfg_dir, cfg) + ["-fPIC", "-shared", "-o", out,
                                                 os.path.join(HERE, "ref_naive_wrap.cpp")])
    return out


def build_ref_sim(name, overrides):
    cfg_dir, cfg = emit_config(name, overrides)
    out = os.path.join(OUT, "TestSimulation_" + name)
    if os.path.exists(out):
        return out
    srcs = [os.path.join(REF, "kernel", f) for f in ("Compute.cpp", "Memory.cpp", "Top.cpp")]
    srcs.append(os.path.join(REF, "test", "TestSimulation.cpp"))
    run(["g++"] + common_flags(cfg_dir, cfg) + ["-o", out] + srcs)
    return out


def build_ref(sim=False):
    if not os.path.isdir(REF):
        return []  # no reference checkout: the tests use the stored outputs under tests/golden/
    os.makedirs(OUT, exist_ok=True)
    jobs = []
    with ThreadPoolExecutor(max_workers=max(1, (os.cpu_count() or 2) - 1)) as ex:
        for name, ov in REF_CONFIGS:
            jobs.append(ex.submit(build_ref_naive, name, ov))
        if sim:
            table = dict(REF_CONFIGS)
            for name in SIM_CONFIGS:
                jobs.append(ex.submit(build_ref_sim, name, table[name]))
        return [j.result() for j in jobs]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref-sim", action="store_true")
    args = ap.parse_args()
    print(build_oracle())
    for p in build_ref(sim=args.ref_sim):
        print(p)


if __name__ == "__main__":
    main()
