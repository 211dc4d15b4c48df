"""The fits predicate that sends a float problem to the f16 wgmma (gemm_hls_b200/csrc/fits_half.h), compiled with g++
and checked against numpy over every TF32 bit pattern of one sign, and the machine code of the float GEMM kernels that
carry both datapaths.  No GPU needed."""
import ctypes
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_sass import CUOBJDUMP, _count, _functions  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "gemm_hls_b200", "csrc", "fits_half.h")

SHIM = r"""
#include "fits_half.h"
extern "C" void fits_all(const uint32_t *bits, unsigned char *out, unsigned count) {
  for (unsigned i = 0; i < count; ++i) out[i] = mm::tf32_fits_half(bits[i]) ? 1 : 0;
}
"""


@pytest.fixture(scope="module")
def fits():
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    d = tempfile.mkdtemp()
    src, lib = os.path.join(d, "shim.cpp"), os.path.join(d, "libshim.so")
    with open(src, "w") as f:
        f.write(SHIM)
    subprocess.run([cxx, "-std=c++17", "-O1", "-shared", "-fPIC", "-I", os.path.dirname(HEADER), src, "-o", lib],
                   check=True)
    so = ctypes.CDLL(lib)

    def run(bits):
        bits = np.ascontiguousarray(bits, dtype=np.uint32)
        out = np.zeros(bits.size, dtype=np.uint8)
        so.fits_all(bits.ctypes.data_as(ctypes.c_void_p), out.ctypes.data_as(ctypes.c_void_p), ctypes.c_uint(bits.size))
        return out.astype(bool)
    yield run
    shutil.rmtree(d, ignore_errors=True)


@pytest.mark.parametrize("sign", [0, 1])
def test_predicate_is_exact_normal_half_round_trip(fits, sign):
    """Every TF32 value (8 exponent + 10 mantissa bits, the low 13 bits zero): the predicate holds exactly when the
    value survives float32 -> float16 -> float32 unchanged as a zero or a normal half.  The one band where a round trip
    also succeeds without the predicate is the half-subnormal range below 2^-14, which the f16 path leaves to TF32."""
    bits = (np.uint32(sign) << np.uint32(31)) | (np.arange(1 << 18, dtype=np.uint32) << np.uint32(13))
    v = bits.view(np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        h = v.astype(np.float16)
        back = h.astype(np.float32)
    exact = (back.view(np.uint32) == bits) & np.isfinite(v)
    normal_or_zero = (h == 0) | (np.abs(h) >= np.float16(2.0 ** -14))
    got = fits(bits)
    assert np.array_equal(got, exact & normal_or_zero)
    assert np.count_nonzero(got) == 30 * 1024 + 1                        # 30 exponents x 1024 mantissas, and the zero
    assert not np.any(got & ~exact)                                      # never a value a half does not hold
    assert np.all((exact & ~got) == (exact & ~normal_or_zero))           # only the half-subnormal band is left out


@pytest.mark.parametrize("sign", [0, 1])
def test_numpy_restatement_matches_the_predicate(fits, sign):
    """tensor_numerics.fits_half_each (on rna_tf32 of its input) against the compiled predicate on every TF32 bit
    pattern of one sign, infinities and NaN included, and on floats whose rounding crosses the boundary."""
    import tensor_numerics as tn
    bits = (np.uint32(sign) << np.uint32(31)) | (np.arange(1 << 18, dtype=np.uint32) << np.uint32(13))
    assert np.array_equal(tn.fits_half_each(bits.view(np.float32)), fits(bits))
    # every float32 just below and above each TF32 value: the predicate of the rounded value
    near = np.concatenate([bits - np.uint32(1), bits + np.uint32(0xFFF), bits + np.uint32(0x1000)])
    near = near[(near >> np.uint32(31)) == sign].view(np.float32)
    with np.errstate(invalid="ignore"):
        rounded = tn.rna_tf32(near).view(np.uint32)
    assert np.array_equal(tn.fits_half_each(near), fits(rounded))
    assert tn.fits_half(np.float32([0.0, -0.0, 9.99, 65504.0])) and not tn.fits_half(np.float32([1.0, 65520.0]))


@pytest.mark.parametrize("x,want", [(0.0, True), (-0.0, True), (2.0 ** -14, True), (2.0 ** -15, False),
                                    (65504.0, True), (65536.0, False), (1e-40, False), (np.inf, False),
                                    (-np.inf, False), (np.nan, False), (9.99, True)])
def test_predicate_boundaries(fits, x, want):
    import tensor_numerics as tn
    assert fits(tn.rna_tf32(np.float32(x)).reshape(1).view(np.uint32))[0] == want


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not installed")
@pytest.mark.parametrize("obj,kernel", [("gemm_tcgen05.o", "gemm_wgmma_kernel"),
                                        ("gemm_wgmma_acc.o", "gemm_wgmma_accumulate_kernel")])
def test_float_kernels_carry_both_datapaths(mm, obj, kernel):
    """Each float (KIND_TF32) wgmma kernel issues TF32 HGMMA and f16 HGMMA (k16, FP32 accumulators), keeps its
    accumulators in registers, and the kernels of the other types are left with their own datapath only."""
    funcs = {k: v for k, v in _functions(obj).items() if kernel in k}
    floats = {k: v for k, v in funcs.items() if "ILi1Ef" in k}
    assert len(floats) == 4                                             # {1, 2 CTAs} x {128, 256 columns}
    for name, ops in floats.items():
        assert _count(ops, "HGMMA") > 0 and all(
            o.split()[0].endswith(".TF32") or ".F32" in o.split()[0] for o in ops if o.startswith("HGMMA")), name
        assert any(o.startswith("HGMMA") and o.split()[0].endswith(".TF32") for o in ops), name
        assert any(o.startswith("HGMMA") and "x16.F32" in o.split()[0] and not o.split()[0].endswith(".TF32")
                   for o in ops), name
        assert _count(ops, "LDL") == 0 and _count(ops, "STL") == 0, name
    for name, ops in funcs.items():
        if name not in floats:
            assert not any(o.startswith("HGMMA") and o.split()[0].endswith(".TF32") for o in ops), name
