"""The bit-packed Boolean restatement (tests/bool_naive.py) against independent oracles, and the GPU test data against
the bugs it must reject; no GPU needed."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bool_naive as bn  # noqa: E402


def brute_product(a, b):
    n, k = a.shape
    m = b.shape[1]
    return np.array([[int(any(a[i, t] and b[t, j] for t in range(k))) for j in range(m)] for i in range(n)], np.uint8)


def test_layout_is_packbits_little():
    x = np.zeros((2, 16), np.uint8)
    x[0, 0] = x[1, 9] = 1
    assert bn.pack(x).tolist() == [[1, 0], [0, 2]]
    assert np.array_equal(bn.unpack(bn.pack(x), 16), x)


@pytest.mark.parametrize("seed", range(4))
def test_product_equals_brute_force(seed):
    a, b = bn.random_bits((7, 19), 0.3, seed), bn.random_bits((19, 11), 0.3, seed + 50)
    assert np.array_equal(bn.product(a, b), brute_product(a, b))


def scipy_closure(d):
    """Reachability by scipy's breadth-first search; the diagonal by the cycle rule: i reaches itself through one or
    more edges iff it has a self-loop or lies in a strongly connected component of two or more vertices."""
    from scipy.sparse import csr_matrix
    from scipy.sparse.csgraph import breadth_first_order, connected_components
    n = d.shape[0]
    g = csr_matrix(d)
    out = np.zeros((n, n), np.uint8)
    for i in range(n):
        out[i, breadth_first_order(g, i, directed=True, return_predecessors=False)] = 1
    _, label = connected_components(g, directed=True, connection="strong")
    size = np.bincount(label)
    np.fill_diagonal(out, ((size[label] > 1) | (np.diag(d) != 0)).astype(np.uint8))
    return out


@pytest.mark.parametrize("graph", ["random", "cycle", "path", "dag", "empty", "complete", "selfloops"])
def test_closure_equals_scipy_and_blocked(graph):
    n = 300
    d = {"random": bn.random_bits((n, n), 0.004, 1), "cycle": bn.hamiltonian_cycle(n, 2), "path": bn.reversed_path(n),
         "dag": bn.random_dag(n, 0.01, 3), "empty": np.zeros((n, n), np.uint8), "complete": np.ones((n, n), np.uint8),
         "selfloops": np.eye(n, dtype=np.uint8)}[graph]
    want = scipy_closure(d)
    assert np.array_equal(bn.closure(d), want)
    for b in (128, 256):  # the block size cannot be seen in the result
        assert np.array_equal(bn.closure_blocked(d, b), want)


# ---- the GPU data rejects plausible bugs -------------------------------------------------------------------------
def test_product_data_rejects_msb_first_bit_order():
    assert any(not np.array_equal(bn.product_msb_first(*bn.product_operands(*c)), bn.product(*bn.product_operands(*c)))
               for c in bn.PRODUCT_CASES)


@pytest.mark.parametrize("stage", [128, 1024])
def test_product_data_rejects_a_dropped_last_chunk_or_stage(stage):
    rejected = 0
    for c in bn.PRODUCT_CASES:
        a, b = bn.product_operands(*c)
        k = a.shape[1]
        if k > stage or stage == 128:
            drop_from = (k - 1) // stage * stage
            rejected += not np.array_equal(bn.product_dropped_k(a, b, drop_from), bn.product(a, b))
    assert rejected >= 2


def test_closure_data_rejects_a_reflexive_diagonal_and_skipped_panels():
    dag = bn.random_dag(1024, 0.002, 11)
    want = bn.closure(dag)
    assert not np.diag(want).any()
    assert not np.array_equal(want | np.eye(1024, dtype=np.uint8), want)
    cyc = bn.hamiltonian_cycle(1024, 12)
    assert not np.array_equal(bn.closure_blocked(cyc, skip_panels=True), bn.closure(cyc))


def test_closure_data_rejects_every_skipped_round():
    cyc = bn.hamiltonian_cycle(1024, 12)  # the GPU test's graph at N = 1024
    want = bn.closure(cyc)
    for r in range(1024 // bn.B):
        assert not np.array_equal(bn.closure_blocked(cyc, skip_round=r), want), r


def test_closure_batch_data_rejects_another_problems_d():
    d = np.stack([bn.random_bits((256, 256), 0.006, 20 + p) for p in range(3)])
    c = [bn.closure(x) for x in d]
    assert all(not np.array_equal(c[p], c[q]) for p in range(3) for q in range(3) if p != q)


# ---- library surface without a GPU -------------------------------------------------------------------------------
def test_null_context_is_invalid(mm):
    L = mm.lib()
    assert L.mm_kernel_enqueue_bool(None, 0, 16, 16, 16, 128, 128, 128, 1, None) == 1
    assert L.mm_kernel_enqueue_bool_closure(None, 0, 16, 128, 1, None) == 1


def test_binding_methods_take_a_context(mm):
    # the entries take an mm_context*: a Multi's handle is an mm_multi*, so the methods live on Context only (one
    # device of a Multi is reached through multi.context(i))
    for name in ("enqueue_bool", "enqueue_bool_closure"):
        assert hasattr(mm.Context, name) and not hasattr(mm.Multi, name), name


def test_library_sass_has_bgmma(mm):
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not installed")
    # the product's object when the build left it (much smaller than the whole library)
    obj = os.path.join(os.path.dirname(mm.LIB_PATH), "build", "gemm_wgmma_b1.o")
    path = obj if os.path.exists(obj) else mm.LIB_PATH
    text = subprocess.run([cuobjdump, "-sass", path], capture_output=True, text=True, check=True).stdout
    assert "BGMMA.64x256x256.AND.POPC" in text and "BGMMA.64x128x256.AND.POPC" in text
