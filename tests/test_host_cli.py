"""The host executables of the reference's CLI surface (SURVEY.md 8b: `TestSimulation N K M`,
`RunHardware.exe N K M [hw|hw_emu] [on|off]`, `PrintSpecifications N K M [MHz]`), built without CMake by
scripts/build_host.sh against the in-tree libmm_b200.so.  CPU checks: usage / shape errors with the
reference's wording and exit codes (host/RunHardware.cpp:41-61), the arithmetic of PrintSpecifications
(src/PrintSpecifications.cpp:16-80), and that a compute call without a GPU fails the way the reference's
runtime errors do (`Execution failed with error: "..."`, exit 1) — there is no CPU fallback."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(tmp, *cfg, static_sizes=None):
    out = str(tmp)
    env = dict(os.environ)
    env.pop("MM_STATIC_SIZES", None)
    if static_sizes:
        env["MM_STATIC_SIZES"] = static_sizes
    r = subprocess.run(["bash", os.path.join(ROOT, "scripts", "build_host.sh"), out, *cfg], capture_output=True, text=True,
                       env=env)
    assert r.returncode == 0, r.stdout + r.stderr
    return out


def _run(exe, *args):
    return subprocess.run([exe, *map(str, args)], capture_output=True, text=True, timeout=120)


@pytest.fixture(scope="module")
def host_float(mm, tmp_path_factory):
    return _build(tmp_path_factory.mktemp("host_float"))


def _field(text, label):
    m = re.search(r"^%s\s+([0-9.e+]+)" % re.escape(label), text, re.M)
    assert m, (label, text)
    return float(m.group(1))


def test_print_specifications_float(host_float):
    r = _run(os.path.join(host_float, "PrintSpecifications"), 16384, 16384, 16384)
    assert r.returncode == 0, r.stderr
    assert "float (Multiply, Add)" in r.stdout and "wgmma_tf32" in r.stdout
    assert _field(r.stdout, "Number of operations:") == pytest.approx(2.0 * 16384 ** 3, rel=1e-5)
    # 132 SMs x 2048 tf32 flop/clk x 1980 MHz
    assert _field(r.stdout, "Ideal performance:") == pytest.approx(132 * 2048 * 1980e-3, rel=1e-4)
    assert _field(r.stdout, "Algorithmic bytes:") == pytest.approx(3 * 4 * 16384 ** 2, rel=1e-5)
    # the reference's I/O model with the CTA-pair tile as memory tile: N*M*(1 + K/256 + K/256) elements
    assert _field(r.stdout, "Communication volume:") == pytest.approx(16384.0 ** 2 * (1 + 64 + 64), rel=1e-5)
    slower = _run(os.path.join(host_float, "PrintSpecifications"), 16384, 16384, 16384, 1000)
    assert _field(slower.stdout, "Ideal performance:") == pytest.approx(132 * 2048 * 1000e-3, rel=1e-4)


def test_print_specifications_uint8_uses_the_integer_tensor_model(mm, tmp_path):
    out = _build(tmp_path, "uint8_t")
    r = _run(os.path.join(out, "PrintSpecifications"), 16384, 16384, 16384)
    assert r.returncode == 0, r.stderr
    assert "uint8_t (Multiply, Add)" in r.stdout and "wgmma_i8" in r.stdout
    # 8-bit wgmma: 132 SMs x 8192 op/clk x 1980 MHz (twice the 16-bit rate)
    assert _field(r.stdout, "Ideal performance:") == pytest.approx(132 * 8192 * 1980e-3, rel=1e-4)


def test_usage_and_shape_errors_follow_the_reference(host_float):
    r = _run(os.path.join(host_float, "PrintSpecifications"))
    assert r.returncode == 1 and "Usage:" in r.stderr
    r = _run(os.path.join(host_float, "RunHardware"), 64, 60, 64, "hw", "on")
    assert r.returncode == 1
    assert "K (60) must be divisable by the memory width in K (16)." in r.stdout + r.stderr
    r = _run(os.path.join(host_float, "RunHardware"), 64, 64, 72)
    assert r.returncode == 1
    assert "M (72) must be divisable by the memory width in M (16)." in r.stdout + r.stderr
    r = _run(os.path.join(host_float, "TestSimulation"), 64, 64)
    assert r.returncode == 1 and "Usage:" in r.stdout + r.stderr


def test_double_model_picks_the_half_height_tile_for_short_row_blocks(mm, tmp_path):
    out = _build(tmp_path, "double")
    full = _run(os.path.join(out, "PrintSpecifications"), 8192, 8192, 8192).stdout
    assert "dmma_f64" in full and "Compute tiles: 128x128 per CTA" in full and "32 waves" in full
    block = _run(os.path.join(out, "PrintSpecifications"), 640, 8192, 8192).stdout  # 320 full tiles = 2.4 waves on 132 SMs
    assert "Compute tiles: 64x128 per CTA" in block and "5 waves" in block


def test_semiring_configuration_reports_the_cuda_core_family(mm, tmp_path):
    out = _build(tmp_path, "float", "Add", "Min")
    text = _run(os.path.join(out, "PrintSpecifications"), 8192, 8192, 8192).stdout
    assert "float (Add, Min)" in text and "semiring_simt" in text
    assert _field(text, "Ideal performance:") == pytest.approx(132 * 128 * 1980e-3, rel=1e-4)


def test_static_size_build_takes_no_shape_arguments(mm, tmp_path):
    """MM_DYNAMIC_SIZES=OFF (CMakeLists.txt:16,43-46 of the reference): N, K, M are compile-time constants."""
    out = _build(tmp_path, static_sizes="1024 2048 512")
    r = _run(os.path.join(out, "PrintSpecifications"))
    assert r.returncode == 0
    assert _field(r.stdout, "Number of operations:") == pytest.approx(2.0 * 1024 * 2048 * 512, rel=1e-5)
    r = _run(os.path.join(out, "PrintSpecifications"), 64, 64, 64)
    assert r.returncode == 1 and "Usage:" in r.stderr and "N K M" not in r.stderr


def test_compute_without_a_gpu_fails_like_a_runtime_error(host_float):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present: the failure path of a missing device cannot be observed")
    for exe, args in (("RunHardware", (64, 64, 64, "hw", "on")), ("TestSimulation", (64, 64, 64))):
        r = _run(os.path.join(host_float, exe), *args)
        assert r.returncode == 1
        assert 'Execution failed with error: "' in r.stdout + r.stderr
