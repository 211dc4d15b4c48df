"""mm_kernel_enqueue_bool and mm_kernel_enqueue_bool_closure on an H100 (run with `-m gpu`): bit for bit against
tests/bool_naive.py and against the library's own uint8 (And, Max) product and closure on the unpacked bytes.

Product: the shapes of bool_naive.PRODUCT_CASES (N 1..1000, K 128..16384, M 128..640, densities from 0.001 to all
ones, and all zeros) into C poisoned with 0xA5 and followed by a 4 KiB guard; a batch of three between two guards;
every tuning variant the kernel honours; graph capture after a sizing call; every validation code.  Closure: a random
Hamiltonian cycle, a reversed path, a DAG, the empty and complete graphs and a random graph at N = 128 .. 4096, a batch
of three, breadth-first reachability at N = 2000 padded to 2048, N = 16384 against repeated squaring through
mm_kernel_enqueue_bool, capture without a prior call, and the new kernels' machine code.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bool_naive as bn  # noqa: E402

pytestmark = pytest.mark.gpu

UINT8, AND, MAX = 5, 4, 3
GUARD = 4096
POISON = 0xA5


@pytest.fixture(scope="module")
def torch():
    t = pytest.importorskip("torch")
    if not t.cuda.is_available():
        pytest.skip("no CUDA device")
    return t


@pytest.fixture(scope="module")
def ctx(mm):
    c = mm.Context(0)
    yield c
    c.close()


class Buf:
    """Bytes on the device between two 4 KiB guards of 0x5A; the body starts 16-byte aligned."""

    def __init__(self, torch, host=None, nbytes=None, fill=POISON):
        self.torch = torch
        self.n = host.size if host is not None else nbytes
        self.buf = torch.full((self.n + 2 * GUARD,), 0x5A, dtype=torch.uint8, device="cuda")
        if host is not None:
            self.buf[GUARD:GUARD + self.n] = torch.from_numpy(np.ascontiguousarray(host).ravel().copy()).cuda()
        else:
            self.buf[GUARD:GUARD + self.n] = fill
        torch.cuda.synchronize()

    @property
    def ptr(self):
        return self.buf.data_ptr() + GUARD

    def result(self):
        self.torch.cuda.synchronize()
        out = self.buf.cpu().numpy()
        assert (out[:GUARD] == 0x5A).all() and (out[GUARD + self.n:] == 0x5A).all(), "a guard changed"
        return out[GUARD:GUARD + self.n]


def gpu_bool(mm, ctx, torch, a, b, batch=1):
    n, k = a.shape[-2:]
    m = b.shape[-1]
    da, db = Buf(torch, bn.pack(a)), Buf(torch, bn.pack(b))
    dc = Buf(torch, nbytes=batch * n * m // 8)
    ctx.enqueue_bool(da.ptr, db.ptr, dc.ptr, n, k, m, batch)
    return bn.unpack(dc.result().reshape(batch, n, m // 8), m).reshape((batch, n, m) if batch > 1 else (n, m))


def uint8_and_max(mm, ctx, torch, a, b):
    n, k = a.shape
    m = b.shape[1]
    da, db, dc = Buf(torch, a), Buf(torch, b), Buf(torch, nbytes=n * m)
    ctx.enqueue(UINT8, AND, MAX, da.ptr, db.ptr, dc.ptr, n, k, m)
    return dc.result().reshape(n, m)


@pytest.mark.parametrize("case", bn.PRODUCT_CASES, ids=["%dx%dx%d-%g" % c[:4] for c in bn.PRODUCT_CASES])
def test_product(mm, ctx, torch, case):
    a, b = bn.product_operands(*case)
    got = gpu_bool(mm, ctx, torch, a, b)
    want = bn.product(a, b)
    assert np.array_equal(got, want)
    assert np.array_equal(got, uint8_and_max(mm, ctx, torch, a, b))


def test_batch_leaves_neighbours_untouched(mm, ctx, torch):
    a = np.stack([bn.random_bits((129, 384), 0.01, 30 + p) for p in range(3)])
    b = np.stack([bn.random_bits((384, 256), 0.01, 40 + p) for p in range(3)])
    got = gpu_bool(mm, ctx, torch, a, b, batch=3)   # Buf checks the guards on both sides
    for p in range(3):
        assert np.array_equal(got[p], bn.product(a[p], b[p])), p


TUNINGS = [dict(cta_group=cg, block_n=bn_, tma_store=ts) for cg in (1, 2) for bn_ in (128, 256) for ts in (0, 1)]
TUNINGS += [dict(stages=2), dict(stages=3, raster_rows=128), dict(tile_sync=0), dict(l2_policy=1), dict(l2_policy=2)]


def test_every_tuning_gives_the_same_bits(mm, torch):
    a, b = bn.product_operands(1000, 1152, 640, 0.01, 50)
    want = bn.product(a, b)
    for t in TUNINGS:
        with mm.Context(0) as c:
            c.set_tuning(**t)
            assert np.array_equal(gpu_bool(mm, c, torch, a, b), want), t


def test_graph_capture_after_a_sizing_call(mm, ctx, torch):
    a, b = bn.product_operands(257, 1152, 384, 0.01, 60)
    want = bn.product(a, b)
    da, db = Buf(torch, bn.pack(a)), Buf(torch, bn.pack(b))
    dc = Buf(torch, nbytes=257 * 384 // 8)
    ctx.enqueue_bool(da.ptr, db.ptr, dc.ptr, 257, 1152, 384)   # sizes the scratch
    dc.result()
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            ctx.enqueue_bool(da.ptr, db.ptr, dc.ptr, 257, 1152, 384, stream=s.cuda_stream)
    for _ in range(2):
        dc.buf[GUARD:GUARD + dc.n] = POISON
        g.replay()
        assert np.array_equal(bn.unpack(dc.result().reshape(257, 48), 384), want)


def test_validation(mm, ctx, torch):
    buf = Buf(torch, nbytes=1 << 20)
    p = buf.ptr
    a, b, c = p, p + (1 << 18), p + (1 << 19)

    def code(fn, *args, **kw):
        with pytest.raises(mm.MMError) as e:
            fn(*args, **kw)
        return e.value.code

    prod, clo = ctx.enqueue_bool, ctx.enqueue_bool_closure
    assert code(prod, None, b, c, 128, 128, 128) == 1
    assert code(prod, a, None, c, 128, 128, 128) == 1
    assert code(prod, a, b, None, 128, 128, 128) == 1
    for n, k, m in ((0, 128, 128), (128, 0, 128), (128, 128, 0)):
        assert code(prod, a, b, c, n, k, m) == 1
    assert code(prod, a, b, c, 128, 64, 128) == 2
    assert code(prod, a, b, c, 128, 128, 192) == 2
    assert code(prod, a, b, c, 128, 128, 128, batch=0) == 1
    assert code(prod, a, b, c, 128, 128, 128, batch=65536) == 5
    assert code(prod, a, b, c, 1 << 20, 128, 128, batch=2048) == 5
    assert code(prod, a + 4, b, c, 128, 128, 128) == 1
    assert code(prod, a, b + 8, c, 128, 128, 128) == 1
    assert code(prod, a, b, c + 1, 128, 128, 128) == 1
    assert code(prod, a, b, c, 128, 128, 128, flags=1) == 1
    assert code(prod, a, b, a + 2048 - 16, 128, 128, 128) == 1   # C's first word is A's last
    assert code(prod, a, b, b - 2048 + 16, 128, 128, 128) == 1   # C's last word is B's first
    prod(a, b, a + 2048, 128, 128, 128)                           # adjacent ranges are accepted
    assert code(clo, None, 128) == 1
    assert code(clo, p, 0) == 1
    assert code(clo, p, 192) == 2
    assert code(clo, p, 128, batch=0) == 1
    assert code(clo, p, 128, batch=65536) == 5
    assert code(clo, p + 16 + 4, 128) == 1
    assert code(clo, p, 128, flags=2) == 1
    buf.result()
    lib = mm.lib()
    assert lib.mm_kernel_enqueue_bool(None, 0, a, b, c, 128, 128, 128, 1, None) == 1
    assert lib.mm_kernel_enqueue_bool_closure(None, 0, p, 128, 1, None) == 1


# ---- closure ----------------------------------------------------------------------------------------------------
def gpu_closure(mm, ctx, torch, d):
    batch, n = (d.shape[0], d.shape[1]) if d.ndim == 3 else (1, d.shape[0])
    dev = Buf(torch, bn.pack(d))
    ctx.enqueue_bool_closure(dev.ptr, n, batch)
    return bn.unpack(dev.result().reshape(d.shape[:-1] + (n // 8,)), n)


def uint8_closure(mm, ctx, torch, d):
    batch, n = (d.shape[0], d.shape[1]) if d.ndim == 3 else (1, d.shape[0])
    dev = Buf(torch, d)
    ctx.enqueue_closure(UINT8, AND, MAX, dev.ptr, n, batch)
    return dev.result().reshape(d.shape)


def graphs(n):
    return {"cycle": bn.hamiltonian_cycle(n, n), "path": bn.reversed_path(n), "dag": bn.random_dag(n, 4.0 / n, n + 1),
            "empty": np.zeros((n, n), np.uint8), "complete": np.ones((n, n), np.uint8),
            "random": bn.random_bits((n, n), 1.0 / n, n + 2)}


@pytest.mark.parametrize("n", [128, 256, 384, 1024, 4096])
def test_closure_against_the_uint8_closure(mm, ctx, torch, n):
    for name, d in graphs(n).items():
        got = gpu_closure(mm, ctx, torch, d)
        assert np.array_equal(got, uint8_closure(mm, ctx, torch, d)), name
        if n <= 1024:
            assert np.array_equal(got, bn.closure(d)), name
        if name == "dag":
            assert not np.diag(got).any()
        if name in ("cycle", "complete"):
            assert got.all()


def test_closure_batch(mm, ctx, torch):
    d = np.stack([bn.random_bits((256, 256), 0.006, 20 + p) for p in range(3)])
    got = gpu_closure(mm, ctx, torch, d)
    assert np.array_equal(got, uint8_closure(mm, ctx, torch, d))
    for p in range(3):
        assert np.array_equal(got[p], bn.closure(d[p])), p


def test_closure_against_bfs_padded(mm, ctx, torch):
    from scipy.sparse import csr_matrix
    from scipy.sparse.csgraph import breadth_first_order
    n, pad = 2000, 2048
    d = bn.random_bits((n, n), 1.2 / n, 77)
    g = csr_matrix(d)
    want = np.zeros((pad, pad), np.uint8)
    for i in range(n):   # paths of one or more edges: one edge, then anything reachable
        for j in np.flatnonzero(d[i]):
            want[i, breadth_first_order(g, j, directed=True, return_predecessors=False)] = 1
    dp = np.zeros((pad, pad), np.uint8)
    dp[:n, :n] = d
    assert np.array_equal(gpu_closure(mm, ctx, torch, dp), want)


def test_closure_at_scale_against_squaring(mm, ctx, torch):
    n = 16384
    with torch.cuda.stream(torch.cuda.Stream()):
        s = torch.cuda.current_stream().cuda_stream
        d = torch.from_numpy(bn.pack(bn.random_bits((n, n), 1.0 / n, 16384))).cuda()
        x = d.clone()
        for _ in range(20):
            y = torch.empty_like(x)
            ctx.enqueue_bool(x.data_ptr(), x.data_ptr(), y.data_ptr(), n, n, n, stream=s)
            y |= x
            if torch.equal(x, y):
                break
            x = y
        assert torch.equal(x, y), "repeated squaring did not reach a fixed point"
        c = d.clone()
        ctx.enqueue_bool_closure(c.data_ptr(), n, stream=s)
        torch.cuda.synchronize()
        assert torch.equal(c, x)


def test_closure_capture_without_a_prior_call(mm, torch):
    d = bn.hamiltonian_cycle(640, 5) | bn.random_bits((640, 640), 0.001, 6)
    want = bn.closure(d)
    with mm.Context(0) as c:
        dev = Buf(torch, bn.pack(d))
        orig = dev.buf.clone()
        s = torch.cuda.Stream()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s):
            torch.cuda.synchronize()
            with torch.cuda.graph(g, stream=s):
                c.enqueue_bool_closure(dev.ptr, 640, stream=s.cuda_stream)
        for _ in range(2):
            dev.buf.copy_(orig)
            g.replay()
            assert np.array_equal(bn.unpack(dev.result().reshape(640, 80), 640), want)


def test_new_kernels_machine_code(mm):
    """BGMMA present and no spills in the Boolean kernels."""
    from test_sass import CUOBJDUMP, _functions
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump not installed")
    bgmma = 0
    for obj in ("gemm_wgmma_b1.o", "bool_closure.o"):
        for name, ops in _functions(obj).items():
            assert not any(o.startswith(("STL", "LDL")) for o in ops), name
            bgmma += sum(1 for o in ops if o.startswith("BGMMA"))
    assert bgmma > 0
