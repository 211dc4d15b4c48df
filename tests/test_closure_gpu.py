"""mm_kernel_enqueue_closure on an H100 (run with `-m gpu`): the closure of every (type, Map, Min | Max) against
tests/closure_naive.py, bit for bit (NaN payload free), on the data of tests/closure_data.py.

Coverage: every pair under MM_FLAG_EXACT and float at flags 0 (FMNMX), at N = 64 (one partial block), b, 2b + w (a
ragged last block) and 3b, and a batch of three at 2b + w.  Every run keeps a 4 KiB guard after D as it was; a call
on the middle problem of three leaves its neighbours untouched.  Independent oracles: float (Add, Min) at N = 2000
against scipy's shortest paths, uint8 (And, Max) reachability against a breadth-first closure, float (Min, Max)
widest paths against thresholded reachability.  Identity traps: float (Multiply, Max) keeps its "no path" zeros;
(Add, Max) on a DAG with negative weights gives the negative longest paths.  Graph capture, validation, and at full
size float and int32 (Add, Min) 8192 against repeated squaring through mm_kernel_enqueue_accumulate to a fixed point.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import closure_data as cd  # noqa: E402
import closure_naive as cn  # noqa: E402
import semiring_data as sd  # noqa: E402
from semiring_data import ADD, AND, FLOAT, INT32, MAX, MIN, MULTIPLY, UINT8  # noqa: E402

pytestmark = pytest.mark.gpu

TA, EXACT, TF32X3, SHARED_A, SHARED_B = 1, 2, 4, 8, 16
GUARD = 4096
PAIRS = [(dt, mp, rd, EXACT) for dt in sd.TYPES for mp in sd.OPS for rd in (MIN, MAX)]
PAIRS += [(FLOAT, mp, rd, 0) for mp in sd.OPS for rd in (MIN, MAX)]


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


def _bytes(x):
    return np.ascontiguousarray(x).view(np.uint8).ravel()


class Dev:
    """D on the device in a buffer with a 4 KiB guard of 0x5A bytes after it."""

    def __init__(self, torch, d):
        self.torch, self.host = torch, np.ascontiguousarray(d)
        raw = _bytes(self.host)
        self.buf = torch.full((raw.size + GUARD,), 0x5A, dtype=torch.uint8, device="cuda")
        self.buf[:raw.size] = torch.from_numpy(raw.copy()).cuda()
        torch.cuda.synchronize()   # the library runs on its context's own stream
        self.n = raw.size

    @property
    def ptr(self):
        return self.buf.data_ptr()

    def result(self):
        self.torch.cuda.synchronize()
        out = self.buf.cpu().numpy()
        assert (out[self.n:] == 0x5A).all(), "the guard after D changed"
        return out[:self.n].view(self.host.dtype).reshape(self.host.shape)


def run(mm, ctx, torch, dt, mp, rd, flags, d):
    batch, n = (d.shape[0], d.shape[1]) if d.ndim == 3 else (1, d.shape[0])
    dev = Dev(torch, d)
    ctx.enqueue_closure(dt, mp, rd, dev.ptr, n, batch, flags)
    return dev.result()


@pytest.mark.parametrize("case", PAIRS, ids=["%s-f%d" % (sd.pair_name(*c[:3]), c[3]) for c in PAIRS])
def test_coverage(mm, ctx, torch, case):
    dt, mp, rd, flags = case
    assert mm.closure_block(dt) == cn.B
    fm = dt == FLOAT and not flags
    w = 64 // sd.SIZE[dt]
    for n, batch in ((64, 1), (128, 1), (2 * 128 + w, 1), (3 * 128, 1), (2 * 128 + w, 3)):
        d = cd.case(dt, mp, rd, n, seed=7, exact=bool(flags), batch=batch)
        want = cn.closure(dt, mp, rd, d, fmnmx=fm)
        got = run(mm, ctx, torch, dt, mp, rd, flags, d if batch > 1 else d[0])
        assert sd.same(got.reshape(want.shape), want), (n, batch)
    # one problem of three: its neighbours stay as they were
    dev = Dev(torch, d)
    es = sd.SIZE[dt]
    ctx.enqueue_closure(dt, mp, rd, dev.ptr + n * n * es, n, 1, flags)
    got = dev.result()
    assert sd.same(got[0], d[0]) and sd.same(got[2], d[2]) and sd.same(got[1], want[1])


def test_nan_term(mm, ctx, torch):
    """A NaN term: the literal Min keeps it, FMNMX drops it."""
    d = cd.case(FLOAT, ADD, MIN, 2 * 128 + 16, seed=5, exact=True, nan_term=True)[0]
    for flags, fm in ((EXACT, False), (0, True)):
        dd = d.copy()
        if fm:   # FMNMX data carries no -0
            dd[dd == 0] = 0.0
        want = cn.closure(FLOAT, ADD, MIN, dd, fmnmx=fm)
        assert sd.same(run(mm, ctx, torch, FLOAT, ADD, MIN, flags, dd), want)


def test_min_plus_against_scipy(mm, ctx, torch):
    csgraph = pytest.importorskip("scipy.sparse.csgraph")
    sparse = pytest.importorskip("scipy.sparse")
    rng = np.random.default_rng(2000)
    n = 2000
    w = rng.integers(1, 100, (n, n)).astype(np.float32)
    absent = rng.random((n, n)) < 0.995
    w[absent] = np.inf
    np.fill_diagonal(w, 0.0)
    g = sparse.csr_matrix(np.where(np.isinf(w), 0, w).astype(np.float64))
    want = csgraph.shortest_path(g, method="D", directed=True)   # weights >= 1: 0 in g is "no edge"
    np.fill_diagonal(want, 0.0)
    for flags in (0, EXACT):
        got = run(mm, ctx, torch, FLOAT, ADD, MIN, flags, w)
        assert np.array_equal(got.astype(np.float64), want)
    assert np.isfinite(want).mean() > 0.5 and want[np.isfinite(want)].max() > 99   # paths of several hops


def _reach(adj):
    """reach[i][j]: a path of >= 1 edge from i to j (repeated boolean squaring, independent of the library)."""
    r = adj.astype(bool)
    while True:
        nxt = r | ((r.astype(np.float32) @ r.astype(np.float32)) > 0)
        if (nxt == r).all():
            return r
        r = nxt


def test_reachability_against_bfs(mm, ctx, torch):
    csgraph = pytest.importorskip("scipy.sparse.csgraph")
    sparse = pytest.importorskip("scipy.sparse")
    rng = np.random.default_rng(512)
    n = 512
    a = (rng.random((n, n)) < 1.2 / n).astype(np.uint8)
    g = sparse.csr_matrix(a)
    reach0 = np.zeros((n, n), np.float32)   # >= 0 edges, by breadth-first search from every vertex
    for s0 in range(n):
        reach0[s0, csgraph.breadth_first_order(g, s0, directed=True, return_predecessors=False)] = 1
    want = (a.astype(np.float32) @ reach0) > 0   # >= 1 edge: a successor, then >= 0 edges
    got = run(mm, ctx, torch, UINT8, AND, MAX, EXACT, a)
    assert np.array_equal(got.astype(bool), want) and set(np.unique(got)) <= {0, 1}
    assert np.array_equal(want, _reach(a))


def test_widest_paths(mm, ctx, torch):
    rng = np.random.default_rng(256)
    n = 2 * 128 + 16
    cap = np.where(rng.random((n, n)) < 3.0 / n, rng.integers(1, 21, (n, n)), 0).astype(np.float32)
    want = np.zeros((n, n), np.float32)
    for t in range(1, 21):   # widest[i][j] = the largest t with a path of edges >= t
        want[_reach(cap >= t)] = t
    got = run(mm, ctx, torch, FLOAT, MIN, MAX, EXACT, cap)
    assert np.array_equal(got, want)
    assert sd.same(got, cn.closure(FLOAT, MIN, MAX, cap))


def test_reliability_keeps_zeros(mm, ctx, torch):
    d = cd.reliability_dag(2 * 128 + 16)
    for flags, fm in ((0, True), (EXACT, False)):
        got = run(mm, ctx, torch, FLOAT, MULTIPLY, MAX, flags, d)
        assert sd.same(got, cn.closure(FLOAT, MULTIPLY, MAX, d, fmnmx=fm))
        assert (got[np.tril_indices(d.shape[0])] == 0).all() and (got[np.triu_indices(d.shape[0], 1)] > 0).mean() > 0.5


def test_longest_paths_on_negative_dag(mm, ctx, torch):
    rng = np.random.default_rng(3)
    n = 3 * 128
    d = np.full((n, n), -np.inf, np.float32)
    iu = np.triu_indices(n, 1)
    keep = rng.random(iu[0].size) < 0.02
    d[iu[0][keep], iu[1][keep]] = rng.integers(-9, 3, keep.sum())
    want = np.full((n, n), -np.inf)
    for j in range(n):   # longest path of >= 1 edge into j, by topological order
        for i in range(j):
            best = d[i, j]
            inner = want[i, i + 1:j] + d[i + 1:j, j]
            want[i, j] = max(best, inner.max()) if inner.size else best
    for flags, fm in ((0, True), (EXACT, False)):
        got = run(mm, ctx, torch, FLOAT, ADD, MAX, flags, d)
        assert np.array_equal(got, want.astype(np.float32))
        assert sd.same(got, cn.closure(FLOAT, ADD, MAX, d, fmnmx=fm))
    assert (want[np.isfinite(want)] < 0).mean() > 0.5


def test_graph_capture(mm, ctx, torch):
    d = cd.case(FLOAT, ADD, MIN, 2 * 128 + 16, seed=9, exact=False)[0]
    direct = run(mm, ctx, torch, FLOAT, ADD, MIN, 0, d)
    dev = Dev(torch, d)
    orig = dev.buf.clone()
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            ctx.enqueue_closure(FLOAT, ADD, MIN, dev.ptr, d.shape[0], 1, 0, stream=s.cuda_stream)
    for _ in range(2):
        dev.buf.copy_(orig)
        g.replay()
        assert sd.same(dev.result(), direct)


def test_validation(mm, ctx, torch):
    dev = Dev(torch, np.zeros((128, 128), np.float32))
    p = dev.ptr

    def code(*args, **kw):
        with pytest.raises(mm.MMError) as e:
            ctx.enqueue_closure(*args, **kw)
        return e.value.code

    assert code(99, ADD, MIN, p, 128) == 1                 # unknown dtype
    assert code(FLOAT, 9, MIN, p, 128) == 1                # unknown map
    assert code(FLOAT, ADD, 9, p, 128) == 1                # unknown reduce
    assert code(FLOAT, ADD, MIN, None, 128) == 1           # null D
    assert code(FLOAT, ADD, MIN, p, 0) == 1                # N = 0
    assert code(FLOAT, ADD, MIN, p, 120) == 2              # N % 16
    assert code(UINT8, AND, MAX, p, 96) == 2               # N % 64
    assert code(FLOAT, ADD, MIN, p, 128, batch=0) == 1
    assert code(FLOAT, ADD, MIN, p, 128, batch=65536) == 5
    assert code(FLOAT, ADD, MIN, p, 1 << 20, batch=2048) == 5   # batch * N >= 2^31
    assert code(FLOAT, ADD, MIN, p + 4, 128) == 1          # misaligned
    assert code(FLOAT, ADD, ADD, p, 128) == 1              # reduce other than Min / Max
    assert code(FLOAT, MULTIPLY, AND, p, 128) == 1
    for f in (TA, SHARED_A, SHARED_B):
        assert code(FLOAT, ADD, MIN, p, 128, flags=f) == 1
    assert mm.closure_block(99) == 0
    d = cd.case(FLOAT, ADD, MIN, 128, seed=1, exact=False)[0]
    assert sd.same(run(mm, ctx, torch, FLOAT, ADD, MIN, TF32X3, d), run(mm, ctx, torch, FLOAT, ADD, MIN, 0, d))


@pytest.mark.parametrize("dt", [FLOAT, INT32])
def test_full_size_against_repeated_squaring(mm, ctx, torch, dt):
    """N = 8192 (Add, Min), integer weights whose path sums stay below 2^24: the closure equals D <- D (+) D (x) D
    through mm_kernel_enqueue_accumulate, repeated to a fixed point (an independent route through existing kernels)."""
    n = 8192
    tdt = torch.float32 if dt == FLOAT else torch.int32
    with torch.cuda.stream(torch.cuda.Stream()):   # a real stream handle: the library and torch order on it
        _full_size(mm, ctx, torch, dt, n, tdt)


def _full_size(mm, ctx, torch, dt, n, tdt):
    gen = torch.Generator(device="cuda").manual_seed(8192)
    d = torch.randint(1, 1000, (n, n), device="cuda", generator=gen, dtype=torch.int32).to(tdt)
    x = d.clone()
    for _ in range(16):
        y = x.clone()
        ctx.enqueue_accumulate(dt, ADD, MIN, x.data_ptr(), x.data_ptr(), y.data_ptr(), n, n, n,
                               stream=torch.cuda.current_stream().cuda_stream)
        if torch.equal(x, y):
            break
        x = y
    assert torch.equal(x, y), "repeated squaring did not reach a fixed point"
    c = d.clone()
    ctx.enqueue_closure(dt, ADD, MIN, c.data_ptr(), n, stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert torch.equal(c.view(torch.int32), x.view(torch.int32))
    assert int(c.max()) < (1 << 24) and bool((c < d).float().mean() > 0.5)   # exact sums; most paths multi-hop


def test_closure_kernels_machine_code(mm):
    """No spills and no FMA contraction in the closure kernels (the checks of tests/test_sass.py), except the
    phase-3 kernels of an And Map on the integer types, which spill as the plain And kernels do (DESIGN.md 3.9)."""
    from test_sass import CUOBJDUMP, _functions, _register_sources
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump not installed")
    seen = 0
    for sfx in ("f16", "f32", "f64", "i32", "u32", "u8", "bf16"):
        for mp in (range(7) if sfx == "f32" else range(5)):
            for name, ops in _functions("semiring_closure_%s_%d.o" % (sfx, mp)).items():
                if "semiring_closure_" not in name:
                    continue
                seen += 1
                bad = [o for o in ops if o.startswith(("FFMA", "DFMA", "HFMA")) and _register_sources(o) >= 3]
                assert not bad, name
                spill = any(o.startswith(("STL", "LDL")) for o in ops)
                allowed = mp == AND and sfx in ("i32", "u32", "u8") and ("ring" in name or "tile" in name)
                assert not spill or allowed, name
    assert seen == 3 * (6 * 5 * 2 + 7 * 4)   # 3 kernels x reduces: (Min, Max) x 5 maps x 6 types; float 7 maps x 4
