"""The reference's two host programs, built from this repo's C++ host mirror (scripts/build_host.sh, no CMake)
and run on the GPU: `TestSimulation N K M` (host pointers through extern "C" MatrixMultiplicationKernel,
test/TestSimulation.cpp:66) and `RunHardware.exe N K M hw on` (Context / Buffer / Kernel, host/RunHardware.cpp).
Both verify against the host ReferenceImplementation with the reference's criterion and print its sentences.
(The file sorts last on purpose: it is the only GPU test that depends on a host compiler at run time.)"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _build(tmp, *cfg, **env):
    if not shutil.which("g++"):
        pytest.skip("no host compiler on this box")
    out = str(tmp)
    r = subprocess.run(["bash", os.path.join(ROOT, "scripts", "build_host.sh"), out, *cfg], capture_output=True, text=True,
                       env=dict(os.environ, **env))
    if r.returncode != 0:
        pytest.skip("host executables did not build here: " + (r.stdout + r.stderr)[-300:])
    return out


def _run(exe, *args, **env):
    return subprocess.run([exe, *map(str, args)], capture_output=True, text=True, timeout=600, env=dict(os.environ, **env))


def test_float_host_programs_verify_on_the_gpu(mm, tmp_path):
    out = _build(tmp_path)
    r = _run(os.path.join(out, "TestSimulation"), 513, 528, 528)        # the reference's CTest shape
    assert r.returncode == 0, r.stdout + r.stderr
    assert "successfully verified" in r.stdout
    r = _run(os.path.join(out, "RunHardware"), 1024, 1024, 1024, "hw", "on")
    assert r.returncode == 0, r.stdout + r.stderr
    assert "Successfully verified." in r.stdout
    m = re.search(r"Kernel executed in ([0-9.e+-]+) seconds, corresponding to a performance of ([0-9.e+-]+) GOp/s", r.stdout)
    assert m, r.stdout                                                   # the line scripts/build_manager.py:601 parses
    assert float(m.group(2)) == pytest.approx(1e-9 * 2.0 * 1024 ** 3 / float(m.group(1)), rel=1e-3)


def test_half_host_programs_take_the_reference_exact_branch(mm, tmp_path):
    """MM_DATA_TYPE=half: the reference compares half results EXACTLY (test/TestSimulation.cpp:79-85) against a
    half-accumulating Naive<>.  The default half build therefore runs the bit-exact datapath and must pass that
    branch at the reference's CTest shape (N = 513, K = 2*32*8 + 32, M = 2*256 + 32)."""
    out = _build(tmp_path, "half")
    r = _run(os.path.join(out, "TestSimulation"), 513, 544, 544)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "successfully verified" in r.stdout
    r = _run(os.path.join(out, "RunHardware"), 256, 256, 256, "hw", "on")
    assert r.returncode == 0 and "Successfully verified." in r.stdout, r.stdout + r.stderr


def test_half_tensor_core_build_verifies_with_fp32_accumulation(mm, tmp_path):
    """-DMM_HALF_TENSOR=ON: half on the tensor cores (FP32 accumulate); the host check uses an FP32-accumulated reference
    and the 1e-3 criterion (INTEGRATION.md section 3 states the deviation from the reference's half-in-half sum)."""
    out = _build(tmp_path, "half", MM_HOST_HALF_TENSOR="1")
    r = _run(os.path.join(out, "TestSimulation"), 513, 544, 544)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "successfully verified" in r.stdout


def test_addmin_and_double_host_programs(mm, tmp_path):
    out = _build(tmp_path / "addmin", "float", "Add", "Min")
    r = _run(os.path.join(out, "TestSimulation"), 513, 528, 528)
    assert r.returncode == 0 and "successfully verified" in r.stdout, r.stdout + r.stderr
    out = _build(tmp_path / "double", "double")
    r = _run(os.path.join(out, "TestSimulation"), 513, 520, 520)
    assert r.returncode == 0 and "successfully verified" in r.stdout, r.stdout + r.stderr


def test_run_hardware_over_mm_num_gpus(mm, tmp_path):
    """MM_NUM_GPUS=2 RunHardware.exe: the row-block split inside the library; with one visible device the request
    fails the way the reference's runtime errors do (message + exit 1) instead of silently shrinking."""
    import torch
    out = _build(tmp_path)
    r = _run(os.path.join(out, "RunHardware"), 1024, 1024, 1024, "hw", "on", MM_NUM_GPUS="2")
    if torch.cuda.device_count() >= 2:
        assert r.returncode == 0 and "Successfully verified." in r.stdout, r.stdout + r.stderr
        assert re.search(r"Kernel executed in [0-9.e+-]+ seconds, corresponding to a performance of [0-9.e+-]+ GOp/s", r.stdout)
    else:
        assert r.returncode == 1 and "Execution failed with error" in r.stderr and "2 devices requested" in r.stderr
