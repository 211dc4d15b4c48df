"""Static checks on the machine code of the accumulate kernels (mm_kernel_enqueue_accumulate), no GPU needed: the
wgmma siblings keep their tensor-core and TMA instructions without spilling, the DMMA siblings keep every FP64 multiply
on the tensor pipe, and no accumulate semiring kernel contracts a Map and a Reduce (or the epilogue's Reduce) into an
FMA.  Same object-file reader and contraction rule as tests/test_sass.py."""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_sass import CUOBJDUMP, _count, _functions, _register_sources  # noqa: E402

pytestmark = pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not installed")

SUFFIXES = ["f16", "f32", "f64", "i32", "u32", "u8", "bf16"]


def test_wgmma_accumulate_kernels(mm):
    funcs = {k: v for k, v in _functions("gemm_wgmma_acc.o").items() if "gemm_wgmma_accumulate_kernel" in k}
    assert len(funcs) == 16                               # {tf32, f16, bf16, u8} x {1, 2 CTAs} x {128, 256 columns}
    for name, ops in funcs.items():
        assert _count(ops, "HGMMA") + _count(ops, "IGMMA") > 0, name
        assert _count(ops, "UTMALDG") > 0 and _count(ops, "UTMASTG") > 0, name
        assert _count(ops, "LDG") > 0, name               # C_old
        assert _count(ops, "LDL") == 0 and _count(ops, "STL") == 0, name
    assert not any("gemm_wgmma_kernel" in k for k in _functions("gemm_wgmma_acc.o"))   # the plain ones stay elsewhere


def test_dmma_accumulate_kernels(mm):
    funcs = {k: v for k, v in _functions("gemm_dmma_acc.o").items() if "gemm_dmma_accumulate_kernel" in k}
    assert len(funcs) == 4                                # {row-major A, A stored K x N} x {128, 64 rows}
    for name, ops in funcs.items():
        assert _count(ops, "DMMA.8x8x4") > 0 and _count(ops, "UTMALDG") > 0, name
        assert _count(ops, "DADD") > 0 and _count(ops, "DFMA") == 0, name
        assert _count(ops, "LDL") == 0 and _count(ops, "STL") == 0, name


@pytest.mark.parametrize("suffix", SUFFIXES)
def test_semiring_accumulate_kernels(mm, suffix):
    maps = range(7) if suffix == "f32" else range(5)
    seen = 0
    for mp in maps:
        funcs = _functions("semiring_accumulate_%s_%d.o" % (suffix, mp))
        assert not any("semiring_tile_kernel" in k or "semiring_ring_kernel" in k for k in funcs)
        for name, ops in funcs.items():
            if "semiring_accumulate_" not in name:
                continue
            seen += 1
            bad = [o for o in ops if o.startswith(("FFMA", "DFMA", "HFMA")) and _register_sources(o) >= 3]
            assert not bad, (name, sorted(set(bad))[:4])
    reduces = 5 * len(maps) + (2 * 7 if suffix == "f32" else 0)   # five reduces per map; FMNMX pairs for float
    assert seen == reduces * (2 if suffix in ("f32", "i32", "u32") else 1)   # 4-byte types: ring and tile kernels
