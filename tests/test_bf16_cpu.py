"""bfloat16 (MM_DTYPE_BFLOAT16) checks that need no GPU: the C-ABI's static queries, the machine code of the
bf16 kernels (cuobjdump on gemm_hls_b200/build/), the bfloat16 Naive<> of tests/bf16_naive.py pinned against an
independent sequential evaluation in torch-CPU bfloat16, and the binding's refusal of float arrays."""
import os
import re
import shutil
import subprocess

import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bf16_naive  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "gemm_hls_b200", "build")
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"

BF16 = 6
MM_ERR_INVALID = 1


# ---- static queries -----------------------------------------------------------------------------

def test_static_queries_of_version_203(mm):
    L = mm.lib()
    assert mm.BFLOAT16 == BF16
    assert L.mm_version() == 203
    assert L.mm_dtype_size(BF16) == 2 and mm.memory_width(BF16) == 32
    assert mm.kernel_path(BF16) == "wgmma_bf16"
    assert mm.launch_count(BF16) == 2                                   # B's K-major copy + GEMM, as half
    assert mm.kernel_path(BF16, flags=mm.FLAG_TRANSPOSED_A) == "wgmma_bf16"
    assert mm.launch_count(BF16, flags=mm.FLAG_TRANSPOSED_A) == 3       # + A's transpose, as half
    assert mm.kernel_path(BF16, flags=mm.FLAG_EXACT) == "semiring_simt"
    assert mm.launch_count(BF16, flags=mm.FLAG_EXACT) == 1
    for mp in range(5):
        for rd in range(5):
            if (mp, rd) != (mm.MULTIPLY, mm.ADD):
                assert mm.kernel_path(BF16, mp, rd) == "semiring_simt", (mp, rd)
                assert mm.launch_count(BF16, mp, rd) == 1, (mp, rd)
    # the 3xTF32 split is float's; bf16 ignores the flag
    assert mm.kernel_path(BF16, flags=mm.FLAG_TF32X3) == "wgmma_bf16"
    assert mm.launch_count(BF16, flags=mm.FLAG_TF32X3) == 2


def test_code_7_is_rejected(mm):
    L = mm.lib()
    assert L.mm_dtype_size(7) == 0 and L.mm_memory_width(7) == 0
    assert mm.kernel_path(7) == "invalid" and mm.launch_count(7) == -1
    buf = np.zeros(64 * 64, dtype=np.uint16)
    p = buf.ctypes.data
    # argument checks come before any device work
    assert L.mm_gemm_host(None, 7, mm.MULTIPLY, mm.ADD, 0, p, p, p, 64, 64, 64, None, None) == MM_ERR_INVALID
    assert "MM_DATA_TYPE" in L.mm_last_error().decode()


def test_binding_refuses_float_arrays_before_device_work(mm):
    ok = np.zeros((32, 32), dtype=np.uint16)
    for bad in (np.zeros((32, 32), dtype=np.float32), np.zeros((32, 32), dtype=np.float16),
                np.zeros((32, 32), dtype=np.float64)):
        with pytest.raises(mm.MMError) as e:
            mm.matrix_multiplication_kernel(bad, ok, 32, 32, 32, dtype=mm.BFLOAT16)
        assert e.value.code == MM_ERR_INVALID and "BFLOAT16" in str(e.value)
        with pytest.raises(mm.MMError) as e:
            mm.matrix_multiplication_kernel(ok, bad, 32, 32, 32, dtype=mm.BFLOAT16)
        assert e.value.code == MM_ERR_INVALID


def test_binding_takes_bit_patterns_by_view(mm):
    x = np.arange(64, dtype=np.uint16).reshape(8, 8)
    v = mm._host_operand(mm.BFLOAT16, x)
    assert v.dtype == np.uint16 and np.shares_memory(v, x)
    ml_dtypes = pytest.importorskip("ml_dtypes")
    y = x.view(ml_dtypes.bfloat16)
    w = mm._host_operand(mm.BFLOAT16, y)
    assert w.dtype == y.dtype and np.shares_memory(w, y)


# ---- machine code ---------------------------------------------------------------------------------

def _functions(obj):
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
    operands = [o.strip() for o in instruction.split(None, 1)[1].split(",")][1:]
    return sum(1 for o in operands if re.match(r"^[-|~]*R\d+", o))


needs_cuobjdump = pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not installed")


@needs_cuobjdump
def test_bf16_gemm_is_wgmma_with_tma(mm):
    funcs = {k: v for k, v in _functions("gemm_wgmma_bf16.o").items() if "gemm_wgmma_kernel" in k}
    assert len(funcs) == 4                                 # {1, 2 CTAs} x {128, 256 columns}
    for name, ops in funcs.items():
        assert any(re.match(r"HGMMA\.\S*BF16", o) for o in ops), name
        assert _count(ops, "UTMALDG") > 0 and _count(ops, "UTMASTG") > 0, name
        assert _count(ops, "HMMA") == 0, name
        assert _count(ops, "LDL") == 0 and _count(ops, "STL") == 0, name
    assert sum(_count(ops, "UTMALDG.2D.MULTICAST") > 0 for ops in funcs.values()) == 2


@needs_cuobjdump
def test_bf16_semiring_kernels_do_not_contract(mm):
    seen = 0
    for mp in range(5):
        for name, ops in _functions("semiring_bf16_%d.o" % mp).items():
            if "semiring_tile_kernel" not in name:
                continue
            seen += 1
            bad = [o for o in ops if o.startswith(("FFMA", "HFMA")) and _register_sources(o) >= 3]
            assert not bad, (name, sorted(set(bad))[:4])
    assert seen >= 25


@needs_cuobjdump
def test_bf16_packed_product_sum_uses_paired_instructions(mm):
    # (Product, Sum): Itanium-mangled 7ProductI...3SumI...
    kern = [ops for name, ops in _functions("semiring_bf16_0.o").items()
            if "semiring_tile_kernel" in name and re.search(r"7Product.*3Sum", name)]
    assert len(kern) == 1
    ops = kern[0]
    # one per pair of C elements, Map and Reduce, per k: 8 rows x 4 pairs x 32 k (one 64-byte k-step) per thread.
    # ptxas spells some of the adds HFMA2.BF16 Rd, Ra, 1, 1, Rb (a * 1 + b: one rounding, no contraction)
    adds = [o for o in ops if o.startswith("HADD2.BF16") or
            (o.startswith(("HFMA2.BF16", "HFMA2.MMA.BF16")) and re.search(r", 1, 1, R\d+$", o))]
    assert _count(ops, "HMUL2.BF16") == 1024 and len(adds) == 1024
    assert _count(ops, "FMUL") == 0 and _count(ops, "FADD") == 0


# ---- the bfloat16 Naive<>, pinned against torch-CPU bfloat16 --------------------------------------------------

@pytest.fixture(scope="module")
def torch():
    return pytest.importorskip("torch")


def _torch_naive(torch, mp, rd, a_bits, b_bits, n, k, m, transposed_a):
    """Naive<> evaluated one k at a time on (n, m) bfloat16 tensors: every Map and every Reduce rounds to bfloat16."""
    bf = torch.bfloat16
    a = torch.from_numpy(a_bits.astype(np.int16).reshape((k, n) if transposed_a else (n, k))).view(bf)
    if transposed_a:
        a = a.t()
    b = torch.from_numpy(b_bits.astype(np.int16).reshape(k, m)).view(bf)

    def bits(v):
        return torch.tensor([v], dtype=torch.int16).view(bf)
    one, zero = bits(0x3F80), bits(0)
    ops = {0: lambda x, y: x * y, 1: lambda x, y: x + y,
           2: lambda x, y: torch.where(x < y, x, y), 3: lambda x, y: torch.where(y < x, x, y),
           4: lambda x, y: torch.where((x != 0) & (y != 0), one, zero)}
    identity = {0: one, 1: zero, 2: bits(0x7F7F), 3: bits(0x0080), 4: one}[rd]
    acc = identity.expand(n, m).clone()
    for kk in range(k):
        acc = ops[rd](acc, ops[mp](a[:, kk:kk + 1], b[kk:kk + 1, :]))
    return acc.contiguous().view(torch.int16).numpy().view(np.uint16)


# bit patterns: NaN, +-0, +-inf, subnormals, the smallest normal, the largest finite value, ordinary values
SPECIAL = np.array([0x7FC0, 0x0000, 0x8000, 0x7F80, 0xFF80, 0x0001, 0x8003, 0x007F, 0x0080, 0x7F7F, 0xFF7F,
                    0x3F80, 0xBF80, 0x4040, 0xC0A0, 0x3E00, 0x0100, 0x8100], dtype=np.uint16)


def _special(rng, size):
    return rng.choice(SPECIAL, size=size).astype(np.uint16)


def _signed(rng, size, scale=2.0):
    x = (rng.standard_normal(size) * scale).astype(np.float32).view(np.uint32)
    return ((x + 0x7FFF + ((x >> 16) & 1)) >> 16).astype(np.uint16)   # float -> bfloat16, to nearest even


@pytest.mark.parametrize("mp", range(5))
@pytest.mark.parametrize("rd", range(5))
def test_bf16_naive_equals_torch_sequential(torch, oracle, mp, rd):
    rng = np.random.default_rng(100 + 5 * mp + rd)
    n, k, m = 9, 64, 32
    a, b = bf16_naive.fill(oracle, n, k, m)
    cases = [("recipe", a, b, n, k, m, False),
             ("signed_ragged", _signed(rng, 37 * 32), _signed(rng, 32 * 32), 37, 32, 32, False),
             ("special", _special(rng, n * k), _special(rng, k * m), n, k, m, False),
             ("transposed", _signed(rng, 13 * 32), _signed(rng, 32 * 64), 13, 32, 64, True)]
    for name, a, b, n, k, m, ta in cases:
        got = bf16_naive.naive(mp, rd, a, b, n, k, m, transposed_a=ta)
        want = _torch_naive(torch, mp, rd, a, b, n, k, m, ta)
        assert got.dtype == np.uint16
        assert bf16_naive.same_nan_free(got, want), name


def test_bf16_fill_is_correctly_rounded(oracle):
    a, b = bf16_naive.fill(oracle, 16, 32, 32)
    ad, bd = oracle.fill(oracle.DOUBLE, 16, 32, 32)    # the same draws, kept in double
    for bits, d in ((a, ad), (b, bd)):
        v = bf16_naive.to_float(bits).astype(np.float64)
        ulp = 2.0 ** (np.floor(np.log2(d)) - 7)
        assert np.all(np.abs(v - d) <= ulp / 2)
        assert np.all((v >= 1.0) & (v <= 10.0))


def test_bf16_double_rounding_is_avoided():
    cases = [(1.0 + 2.0 ** -8, 0x3F80),                  # tie: to even (down)
             (1.0 + 3 * 2.0 ** -8, 0x3F82),              # tie: to even (up)
             (1.0 + 2.0 ** -8 + 2.0 ** -40, 0x3F81),     # just above the tie: through float32 it would become the tie
             (-(1.0 + 2.0 ** -8 + 2.0 ** -40), 0xBF81),
             (2.0 ** 128 - 2.0 ** 119, 0x7F80),          # half an ulp above the largest finite value: to infinity
             (2.0 ** 128 - 2.0 ** 119 - 2.0 ** 100, 0x7F7F),
             (2.0 ** -133, 0x0001), (2.0 ** -134, 0x0000), (1.5 * 2.0 ** -133, 0x0002),   # subnormals, ties to even
             (0.0, 0x0000), (-0.0, 0x8000), (float("inf"), 0x7F80), (float("-inf"), 0xFF80)]
    for d, want in cases:
        assert int(bf16_naive.from_double(np.array([d]))[0]) == want, (d, want)
    assert (int(bf16_naive.from_double(np.array([float("nan")]))[0]) & 0x7FFF) > 0x7F80


def test_bf16_naive_identities():
    # K = 0 is not a legal shape for the product, but Naive<> returns the Reduce identity for it
    for rd, want in ((0, 0x3F80), (1, 0x0000), (2, 0x7F7F), (3, 0x0080), (4, 0x3F80)):
        c = bf16_naive.naive(bf16_naive.ADD, rd, np.zeros(0, np.uint16), np.zeros(0, np.uint16), 4, 0, 32)
        assert c.shape == (4, 32) and np.all(c == want), rd
