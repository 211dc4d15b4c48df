#!/usr/bin/env python
"""Build gemm_hls_b200/libmm_b200.so (the C-ABI library, include/mm_b200.h) for sm_90a with nvcc.

    python gemm_hls_b200/build.py [--force] [--verbose]

Objects go to gemm_hls_b200/build/ (git-ignored); the .so stays in-tree next to this file, where the
Python binding loads it.  nvcc cross-compiles without a GPU.
"""
import argparse
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libmm_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
         "--expt-relaxed-constexpr"]

SOURCES = ["capi.cu", "gemm_tcgen05.cu", "gemm_wgmma_bf16.cu", "gemm_wgmma_acc.cu", "gemm_dmma.cu", "gemm_dmma_acc.cu",
           "semiring_dispatch.cu", "gemm_wgmma_b1.cu", "bool_closure.cu"]
# semiring_inst.cu, semiring_witness_inst.cu, semiring_accumulate_inst.cu and semiring_closure_inst.cu are compiled
# once per (type, map operator): (object suffix, C type)
INST_TYPES = [("f16", "__half"), ("f32", "float"), ("f64", "double"), ("i32", "int"),
              ("u32", "unsigned"), ("u8", "unsigned char"),
              ("bf16", "__nv_bfloat16")]
INST_MAPS = [0, 1, 2, 3, 4]  # MM_OP_MULTIPLY .. MM_OP_AND


def newest_header():
    t = 0.0
    for d in (CSRC, os.path.join(HERE, "..", "include")):
        for f in os.listdir(d):
            if f.endswith((".cuh", ".h")):
                t = max(t, os.path.getmtime(os.path.join(d, f)))
    return t


def compile_one(job, force, verbose, hdr_time):
    src, objname, defines = job
    s = os.path.join(CSRC, src)
    o = os.path.join(OBJ, objname)
    if not force and os.path.exists(o) and os.path.getmtime(o) >= max(os.path.getmtime(s), hdr_time):
        return o, False
    cmd = [NVCC] + ARCH + FLAGS + defines + (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout[-4000:] + r.stderr[-8000:])
        raise RuntimeError("nvcc failed on " + src)
    if verbose:
        sys.stderr.write(r.stderr)
    return o, True


def newest_source():
    return max(os.path.getmtime(os.path.join(CSRC, f)) for f in os.listdir(CSRC) if f.endswith(".cu"))


def build(force=False, verbose=False):
    hdr_time = newest_header()
    # An up-to-date library needs nothing, even where the objects it was linked from were left behind
    # (a copy of the tree made to run it elsewhere need not carry gemm_hls_b200/build/).
    if not force and not verbose and os.path.exists(LIB) and os.path.getmtime(LIB) >= max(hdr_time, newest_source()):
        return LIB
    os.makedirs(OBJ, exist_ok=True)
    with ThreadPoolExecutor(max_workers=max(1, (os.cpu_count() or 2))) as ex:
        jobs = [(src, obj % (suffix, mp), ["-DMM_INST_T=" + ctype, "-DMM_INST_MAP=%d" % mp])
                for src, obj in (("semiring_inst.cu", "semiring_%s_%d.o"),
                                 ("semiring_witness_inst.cu", "semiring_witness_%s_%d.o"),
                                 ("semiring_accumulate_inst.cu", "semiring_accumulate_%s_%d.o"),
                                 ("semiring_closure_inst.cu", "semiring_closure_%s_%d.o"))
                for suffix, ctype in INST_TYPES for mp in INST_MAPS + ([5, 6] if suffix == "f32" else [])]
        jobs += [(src, src.replace(".cu", ".o"), []) for src in SOURCES]
        results = list(ex.map(lambda j: compile_one(j, force, verbose, hdr_time), jobs))
    objs = [o for o, _ in results]
    if any(changed for _, changed in results) or not os.path.exists(LIB):
        cmd = [NVCC] + ARCH + ["-shared", "-o", LIB] + objs + ["-Xlinker", "--exclude-libs=ALL"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    return LIB


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--verbose", action="store_true")
    a = ap.parse_args()
    print(build(a.force, a.verbose))
