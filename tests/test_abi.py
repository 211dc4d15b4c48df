"""CPU tests of the drop-in boundary: libmm_b200.so loads and exports every symbol that
include/mm_b200.h declares; argument validation and error reporting work without a GPU; and the
product refuses to compute when no CUDA device is present (no CPU fallback)."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "mm_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(mm_[a-z0-9_]+)\s*\(", text)))


def test_header_symbols_are_exported(mm):
    syms = declared_symbols()
    assert len(syms) >= 15
    L = ctypes.CDLL(mm.LIB_PATH)
    for s in syms:
        assert hasattr(L, s), "libmm_b200.so does not export " + s
    assert set(syms) == set(mm.EXPORTS)


def test_only_the_c_abi_is_exported(mm):
    out = subprocess.run(["nm", "-D", "--defined-only", mm.LIB_PATH], capture_output=True, text=True).stdout
    exported = [l.split()[-1] for l in out.splitlines() if " T " in l]
    assert exported and all(s.startswith("mm_") for s in exported), exported


def test_library_contains_hopper_sass(mm):
    """wgmma / TMA must be in the shipped cubin: HGMMA / IGMMA (wgmma.mma_async), UTMALDG / UTMASTG
    (cp.async.bulk.tensor), DMMA (the double path)."""
    r = subprocess.run(["cuobjdump", "-sass", mm.LIB_PATH], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("cuobjdump not available")
    sass = r.stdout
    assert "sm_90a" in sass and "sm_100" not in sass
    assert "HGMMA" in sass, "no wgmma.mma_async in SASS"
    assert "IGMMA" in sass, "no integer wgmma (u8) in SASS"
    assert "UTMALDG" in sass
    assert "UTMASTG" in sass, "the epilogue's TMA stores are missing"
    assert "DMMA" in sass


def test_static_queries(mm):
    assert mm.lib().mm_version() >= 200
    assert [mm.lib().mm_dtype_size(d) for d in range(6)] == [2, 4, 8, 4, 4, 1]
    assert mm.memory_width(mm.FLOAT) == 16 and mm.memory_width(mm.HALF) == 32
    assert mm.memory_width(mm.DOUBLE) == 8 and mm.memory_width(mm.UINT8) == 64
    assert mm.kernel_path(mm.FLOAT) == "wgmma_tf32"
    assert mm.kernel_path(mm.HALF) == "wgmma_f16"
    assert mm.kernel_path(mm.DOUBLE) == "dmma_f64"
    assert mm.kernel_path(mm.FLOAT, mm.ADD, mm.MIN) == "semiring_simt"
    assert mm.kernel_path(mm.FLOAT, flags=mm.FLAG_EXACT) == "semiring_simt"
    assert mm.kernel_path(mm.INT32) == "semiring_simt"
    assert mm.kernel_path(mm.UINT8) == "wgmma_i8" and mm.kernel_path(mm.UINT8, flags=mm.FLAG_EXACT) == "semiring_simt"
    assert mm.kernel_path(mm.UINT8, mm.ADD, mm.MIN) == "semiring_simt" and mm.launch_count(mm.UINT8, mm.ADD, mm.MIN) == 1
    # float: B rounding + A rounding + GEMM; half and uint8_t read A in place and B from its K-major copy
    assert mm.launch_count(mm.FLOAT) == 3 and mm.launch_count(mm.DOUBLE) == 1
    assert mm.launch_count(mm.HALF) == 2 and mm.launch_count(mm.UINT8) == 2


def test_multi_partition_rule_needs_no_device(mm):
    """mm_multi_partition: the cut every mm_multi_* entry applies (rows of A / C, K-row slices of B in multiples of 64)."""
    for n, k, g_count in ((16384, 16384, 8), (513, 528, 3), (3, 64, 4), (8192, 8192, 1), (100, 4096, 7)):
        rows, slices = [], []
        for g in range(g_count):
            r0, r1, k0, k1 = mm.multi_partition(g_count, g, n, k)
            assert 0 <= r0 <= r1 <= n and 0 <= k0 <= k1 <= k
            assert (k0 % 64 == 0 and ((k1 - k0) % 64 == 0 or k1 == k)) or g_count == 1
            rows.append((r0, r1))
            slices.append((k0, k1))
        assert rows[0][0] == 0 and slices[0][0] == 0
        assert sum(b - a for a, b in rows) == n and sum(b - a for a, b in slices) == k
        for (a0, a1), (b0, b1) in zip(rows, rows[1:]):
            assert a1 == b0
        for (a0, a1), (b0, b1) in zip(slices, slices[1:]):
            assert a1 == b0
    assert mm.multi_partition(8, 5, 16384, 16384) == (10240, 12288, 10240, 12288)
    assert mm.multi_partition(4, 3, 3, 64) == (3, 3, 64, 64)          # more GPUs than rows and than slices
    with pytest.raises(mm.MMError):
        mm.multi_partition(2, 2, 10, 64)


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def test_argument_validation_before_any_device_work(mm):
    a = np.ones(16 * 16, dtype=np.float32)
    with pytest.raises(mm.MMError) as e:
        mm.matrix_multiplication_kernel(a, a, 16, 16, 16, dtype=99)
    assert e.value.code == 1
    with pytest.raises(mm.MMError) as e:  # K not a multiple of the 64-byte memory word
        mm.matrix_multiplication_kernel(np.ones(16 * 24, np.float32), np.ones(24 * 16, np.float32), 16, 24, 16)
    assert e.value.code == 2 and "divisable by the memory width in K" in str(e.value)
    with pytest.raises(mm.MMError) as e:
        mm.matrix_multiplication_kernel(np.ones(16 * 16, np.float32), np.ones(16 * 8, np.float32), 16, 16, 8)
    assert e.value.code == 2 and "memory width in M" in str(e.value)


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU behaviour")
def test_no_cpu_fallback_without_a_gpu(mm):
    """Without a CUDA device the compute entry points fail loudly (MM_ERR_CUDA = 3)."""
    a = np.ones(16 * 16, dtype=np.float32)
    with pytest.raises(mm.MMError) as e:
        mm.matrix_multiplication_kernel(a, a, 16, 16, 16)
    assert e.value.code == 3
    with pytest.raises(mm.MMError) as e:
        mm.Context(0)
    assert e.value.code == 3
