"""bench.py's driver contract, as far as it can be exercised without a GPU: the reference arm
(`--impl reference`: the reference's own Naive<> on the host cores) prints one JSON line with the agreed
keys, non-zero ranks of a torchrun launch stay silent, and the GPU arm refuses to run without a device
(no CPU fallback on the product path)."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _bench(*args, env=None):
    e = dict(os.environ)
    e.update(env or {})
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), *args], capture_output=True, text=True,
                          timeout=600, env=e, cwd=ROOT)


def test_reference_arm_line(oracle):
    r = _bench("--impl", "reference", "--workload", "float4096", "--steps", "2", "--warmup", "1")
    assert r.returncode == 0, r.stderr
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["n_gpus"] == 1 and d["steps"] == 2 and d["warmup"] >= 3
    assert d["unit"] == "GFLOP/s" and d["higher_is_better"] is True and d["gpu_launches"] == 0
    assert d["metric"].startswith("GFLOP/s at N=4096 K=4096 M=4096 float")
    assert d["value"] > 0 and d["ms_per_step"] > 0
    cb = d["cpu_baseline"]
    assert cb["kind"] in ("reference", "port") and cb["cores"] >= 1 and cb["value"] == d["value"]
    assert "Naive<>" in cb["sample"]
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    # value = sampled operations / time: rows x K x sampled columns x 2 per step; the sample is FIXED
    # (one row per physical core, first SAMPLE_COLS columns), never shrunk adaptively
    import bench
    rows = int(cb["sample"].split()[0])
    assert rows == cb["cores"] == bench.host_threads()
    assert d["value"] == pytest.approx(1e-9 * 2.0 * rows * 4096 * bench.SAMPLE_COLS / (1e-3 * d["ms_per_step"]), rel=1e-6)
    # both arms print the same `config` (nothing run-dependent in it): the driver's same_config check
    assert set(d["config"]) == {"workload", "baseline_config", "partition", "l2"}


def test_reference_arm_runs_on_rank_zero_only(oracle):
    r = _bench("--impl", "reference", "--workload", "float4096", "--steps", "1", "--gpus", "2",
               env={"RANK": "1", "LOCAL_RANK": "1", "WORLD_SIZE": "2"})
    assert r.returncode == 0 and r.stdout.strip() == ""


def test_b200_arm_has_no_cpu_fallback(mm):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    r = _bench("--workload", "float4096", "--steps", "1")
    assert r.returncode != 0
    assert "no CPU fallback" in r.stderr + r.stdout


def test_cpu_baseline_object_of_the_b200_arm(oracle):
    """The helper the GPU arm calls with host copies of its device inputs (no GPU needed to run it)."""
    import numpy as np
    sys.path.insert(0, ROOT)
    import bench
    k = m = 512
    rng = np.random.default_rng(1)
    a = rng.uniform(1, 10, size=(64, k)).astype(np.float32)
    b = rng.uniform(1, 10, size=(k, m)).astype(np.float32)
    asked = []

    def a_rows_of(rows):
        asked.append(rows)
        return a[:min(rows, a.shape[0])]

    cb = bench.cpu_baseline_line("float", "Multiply", "Add", "GFLOP/s", k, m, a_rows_of, b)
    threads = bench.host_threads()
    assert asked == [threads]                         # one row per physical core, as in the reference arm
    rows = min(threads, 64)
    assert cb["cores"] == min(threads, rows) and cb["kind"] in ("reference", "port") and cb["unit"] == "GFLOP/s"
    assert cb["value"] == pytest.approx(1e-9 * 2.0 * rows * k * min(m, bench.SAMPLE_COLS) / cb["seconds"], rel=1e-9)
    assert cb["sample"].startswith("%d rows x first %d columns of C" % (rows, min(m, bench.SAMPLE_COLS)))


def test_numa_placed_host_matrix_helper_without_a_gpu():
    """bench.alloc_host_rows, several blocks: an anonymous mapping, each row-block first-touched by its own thread, then
    registered (here with a stand-in for cudart).  Without NVML / sysfs the placement degrades to 'no affinity'."""
    import types

    import numpy as np
    import bench
    calls = []

    class FakeRuntime:
        def cudaHostRegister(self, ptr, nbytes, flags):
            calls.append((ptr, nbytes, flags))
            return 0

    fake_torch = types.SimpleNamespace(cuda=types.SimpleNamespace(cudart=lambda: FakeRuntime()))
    arr, keep, note = bench.alloc_host_rows(fake_torch, 1000, 64, np.float32, [(0, 500, 0), (500, 1000, 1)])
    assert arr.shape == (1000, 64) and arr.dtype == np.float32 and arr.flags["C_CONTIGUOUS"] and arr.flags["WRITEABLE"]
    assert calls == [(arr.ctypes.data, 1000 * 64 * 4, 0)] and keep is not None
    assert note.startswith("registered page-locked") and not arr.any()
    arr[:] = 3.0
    assert float(arr.sum()) == 3.0 * 64000
    assert bench.node_cpus(10 ** 6) == set()       # a node that does not exist
