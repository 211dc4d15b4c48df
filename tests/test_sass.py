"""Static checks on the machine code of the built kernels (cuobjdump on the objects of
gemm_hls_b200/build/, no GPU needed): the Hopper (sm_90a) instructions each path claims are there, and —
the part that protects bit-exactness — ptxas has not contracted a multiply and an add into an FMA anywhere in
the float / double / half semiring kernels (Naive<> rounds after the Map and again after the Reduce)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "gemm_hls_b200", "build")
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"

pytestmark = pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not installed")


def _functions(obj):
    """{mangled function name: [instruction text, ...]} of one object file ("FADD2 R60, R88.F32, ...")."""
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
        m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][^;]*);", line)
        if m and name:
            funcs[name].append(m.group(1).strip())
    return funcs


def _count(ops, prefix):
    return sum(1 for o in ops if o.startswith(prefix))


def _register_sources(instruction):
    """Number of source operands that are real registers (not RZ, not immediates)."""
    operands = [o.strip() for o in instruction.split(None, 1)[1].split(",")][1:]
    return sum(1 for o in operands if re.match(r"^[-|~]*R\d+", o))


def test_tensor_core_gemm_is_wgmma_with_tma(mm):
    funcs = {k: v for k, v in _functions("gemm_tcgen05.o").items() if "gemm_wgmma_kernel" in k}
    assert funcs
    for name, ops in funcs.items():
        assert _count(ops, "HGMMA") + _count(ops, "IGMMA") > 0, name   # wgmma.mma_async (tf32 / f16 | u8)
        assert _count(ops, "UTMALDG") > 0, name          # cp.async.bulk.tensor loads
        assert _count(ops, "UTMASTG") > 0, name          # cp.async.bulk.tensor stores (the epilogue)
        assert _count(ops, "HMMA") == 0 and _count(ops, "IMMA") == 0, name    # no warp-level mma.sync path
        assert _count(ops, "LDL") == 0 and _count(ops, "STL") == 0, name      # accumulators stay in registers
    assert sum(_count(ops, "HGMMA.64x256x8.F32.TF32") > 0 for ops in funcs.values()) == 2   # float, 1 and 2 CTAs
    assert any(_count(ops, "IGMMA.64x256x32.U8.U8") > 0 for ops in funcs.values())          # uint8_t, exact s32
    assert sum(_count(ops, "UTMALDG.2D.MULTICAST") > 0 for ops in funcs.values()) == 6      # cluster variants share B
    assert len(funcs) == 12                               # {tf32, f16, u8} x {1, 2 CTAs} x {128, 256 columns}


def test_double_gemm_is_dmma_fed_by_tma_without_ldgsts(mm):
    funcs = {k: v for k, v in _functions("gemm_dmma.o").items() if "gemm_dmma_tma_kernel" in k}
    assert len(funcs) == 4                                # {row-major A, A stored K x N} x {128, 64 rows}
    for name, ops in funcs.items():
        assert _count(ops, "DMMA.8x8x4") > 0 and _count(ops, "UTMALDG") > 0, name
        assert _count(ops, "LDGSTS") == 0, name           # the loads are TMA, not cp.async
        assert _count(ops, "LDL") == 0 and _count(ops, "STL") == 0, name      # no spills
        assert _count(ops, "DFMA") == 0, name             # all FP64 math on the tensor pipe


def _semiring(obj, mp, rd, kernel="semiring_tile_kernel"):
    """The kernel for (Map, Reduce) in a semiring object; names are Itanium-mangled (3Sum, 7Product, ...)."""
    tag = {"Sum": "3Sum", "Product": "7Product", "Min": "3Min", "Max": "3Max", "And": "3And",
           "MinFast": "7MinFast", "MaxFast": "7MaxFast"}
    out = []
    for name, ops in _functions(obj).items():
        if kernel not in name:
            continue
        m = re.search(kernel + r"I\w(?:NS_)?(\d[A-Za-z]+)I\w+?E(?:NS_(\d[A-Za-z]+)I\w+?E|(S\d?_))", name)
        assert m, name
        mapped = m.group(1)
        reduced = m.group(2) if m.group(2) else mapped   # a substitution (S2_) repeats the Map type
        if mapped == tag[mp] and reduced == tag[rd]:
            out.append((name, ops))
    assert len(out) == 1, (obj, mp, rd, [n for n, _ in out])
    return out[0][1]


def test_float_semiring_inner_loops(mm):
    """One Map and one Reduce instruction per element and k step: 8 x 8 elements x 16 k per unrolled tile."""
    addmin = _semiring("semiring_f32_1.o", "Sum", "MinFast")
    assert _count(addmin, "FADD") == 1024 and _count(addmin, "FMNMX") == 1024
    assert _count(addmin, "UTMALDG") > 0                                           # B tile staged by TMA
    ring = _semiring("semiring_f32_1.o", "Sum", "MinFast", kernel="semiring_ring_kernel")  # the default for 4-byte types
    assert _count(ring, "FADD") == 1024 and _count(ring, "FMNMX") == 1024
    assert _count(ring, "UTMALDG") >= 2 and _count(ring, "LDG") == 0 and _count(ring, "BAR") <= 2   # both tiles by TMA, no barrier in the loop
    exact = _semiring("semiring_f32_0.o", "Product", "Sum")
    assert _count(exact, "FMUL") == 1024 and _count(exact, "FADD") == 1024 and _count(exact, "FFMA") == 0


@pytest.mark.parametrize("suffix", ["f32", "f64", "f16"])
def test_no_fma_contraction_in_any_floating_point_semiring_kernel(mm, suffix):
    seen = 0
    for mp in range(5):
        for name, ops in _functions("semiring_%s_%d.o" % (suffix, mp)).items():
            if "semiring_tile_kernel" not in name and "semiring_ring_kernel" not in name:
                continue
            seen += 1
            # a contraction multiplies two data registers and adds a third.  What may legitimately appear:
            # HFMA2 Rd, -RZ, RZ, imm, imm (constant materialisation) and HFMA2 Rd, Ra, 1, 1, Rb (the
            # compiler's spelling of a half ADD: a * 1 + b, one rounding)
            bad = [o for o in ops if o.startswith(("FFMA", "DFMA", "HFMA")) and _register_sources(o) >= 3]
            assert not bad, (name, sorted(set(bad))[:4])
    assert seen >= 25


def test_the_contraction_detector_itself():
    assert _register_sources("FFMA2 R2, R100.F32, R104.reuse.F32x2.HI_LO, R60.F32x2.HI_LO") == 3   # what ptxas made of mul+add
    assert _register_sources("FFMA R4, R5, R6, R4") == 3
    assert _register_sources("HFMA2 R93, -RZ, RZ, 1.984375, 0") == 0                               # constant
    assert _register_sources("HFMA2 R7, R7, 1, 1, R9") == 2                                        # half add
    assert _register_sources("FMUL2 R8, R2.F32, R4.F32x2.HI_LO") == 2
