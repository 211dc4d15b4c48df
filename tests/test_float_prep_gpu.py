"""The float operand preparation writes one copy per 64 x 64 item (run with `-m gpu` on an H100).

A float problem reads either the TF32 copies of its operands or their fp16 copies.  The first preparation pass writes
the fp16 copy of an item until a fits word that already reads 0 proves that every problem reading the copy runs on
TF32; from then on it writes the TF32 copy.  A second pass, once the words are final, writes the TF32 copies still
owed (one pending byte per item).  What the datapath tests cannot see is a stale copy: an item that neither pass wrote
in this call, read from an earlier call.  So every call here takes fresh data, and each C must equal, bit for bit, the
same call in a fresh context; a problem that runs on TF32 must also equal the tf32_no_round call on the same
(TF32-exact) data, which prepares its operands by another route.

Data kinds, on fp16-exact U[1, 10) (rounding to TF32 is the identity):
  fit     every value a normal half: f16 datapath
  early   B[0, 0] = 2^16: the first item of the pass does not fit, nearly every other item settles on TF32
  late    A[N-1, K-1] = 2^16: the last item does not fit, every other item was prepared as fp16 and is owed as TF32
"""
import itertools
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_float_datapaths_gpu as fdg  # noqa: E402
import test_tensor_numerics_gpu as tng  # noqa: E402

pytestmark = pytest.mark.gpu

N = K = M = 2048          # 1024 items per operand: more than the persistent grid has blocks (132 SMs x 8)
KINDS = ("fit", "early", "late")
NOT_HALF = np.float32(2.0 ** 16)   # TF32-exact, not a half


@pytest.fixture(scope="module")
def torch():
    t = pytest.importorskip("torch")
    if not t.cuda.is_available():
        pytest.skip("no CUDA device")
    return t


def operands(kind, seed, n=N, k=K, m=M):
    a, b = fdg.probe_operands(n, k, m, seed=seed)
    a, b = a[0], b[0]
    if kind == "early":
        b[0, 0] = NOT_HALF
    elif kind == "late":
        a[n - 1, k - 1] = NOT_HALF
    return a, b


def run(torch, mm, ctx, a, b, n=N, k=K, m=M):
    return tng._run(torch, mm, ctx, "tf32", tng._dev(torch, "tf32", a), tng._dev(torch, "tf32", b), n, k, m)


def fresh(torch, mm, a, b, n=N, k=K, m=M, **knobs):
    return fdg._call(torch, mm, knobs, a, b, n, k, m)


def check(torch, mm, got, a, b, kind, what, n=N, k=K, m=M):
    assert fdg.same_bits(got, fresh(torch, mm, a, b, n, k, m)), what
    tf32 = fresh(torch, mm, a, b, n, k, m, tf32_no_round=1)
    if kind == "fit":
        assert fdg.classify(got, tf32) == "tf32h", what
    else:
        assert fdg.same_bits(got, tf32), what


@pytest.mark.parametrize("first,second", list(itertools.product(KINDS, KINDS)))
def test_sequence_in_one_context(torch, mm, first, second):
    data = [operands(first, 11), operands(second, 12)]
    with mm.Context(0) as ctx:
        got = [run(torch, mm, ctx, *data[0]), run(torch, mm, ctx, *data[1])]
    for i, kind in enumerate((first, second)):
        check(torch, mm, got[i], *data[i], kind, (first, second, i))


def test_sequence_under_graph_replay(torch, mm):
    """One captured call replayed over fresh contents of every kind; the sequence holds every ordered pair."""
    seq = ["fit", "fit", "early", "early", "late", "late", "fit", "late", "early", "fit"]
    a0, b0 = operands("fit", 0)
    da, db = tng._dev(torch, "tf32", a0), tng._dev(torch, "tf32", b0)
    c = torch.empty((N * M,), dtype=torch.float32, device="cuda")
    with mm.Context(0) as ctx:
        ctx.reserve(mm.FLOAT, N, K, M)
        s = torch.cuda.Stream()
        g = torch.cuda.CUDAGraph()
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            ctx.enqueue(mm.FLOAT, mm.MULTIPLY, mm.ADD, da.data_ptr(), db.data_ptr(), c.data_ptr(), N, K, M,
                        stream=s.cuda_stream)
        for i, kind in enumerate(seq):
            a, b = operands(kind, 100 + i)
            da.copy_(torch.from_numpy(a))
            db.copy_(torch.from_numpy(b))
            c.fill_(float("nan"))
            torch.cuda.synchronize()
            g.replay()
            torch.cuda.synchronize()
            check(torch, mm, c.cpu().numpy().reshape(N, M), a, b, kind, (i, kind))
        del g


@pytest.mark.parametrize("which", ["a", "b"])
def test_partner_settling(torch, mm, which):
    """One operand does not fit from its first item; the other fits, and its items settle on its partner's word."""
    with mm.Context(0) as ctx:
        run(torch, mm, ctx, *operands("fit", 20))     # leaves fp16 copies of other data behind
        a, b = operands("fit", 21)
        if which == "a":
            a[0, 0] = NOT_HALF
        else:
            b[0, 0] = NOT_HALF
        got = run(torch, mm, ctx, a, b)
    check(torch, mm, got, a, b, "no fit", which)


def test_shared_a_keeps_its_fp16_copy(torch, mm):
    """A batch with a shared A: problem 0's B does not fit from its first item, problem 1's fits.  The shared A must
    not settle on problem 0's word: problem 1 runs on f16 and reads A's fp16 copy."""
    n = k = m = 1024
    rng = np.random.default_rng(30)
    with mm.Context(0) as ctx:
        for seed in (31, 32):
            a = rng.uniform(1, 10, (1, n, k)).astype(np.float16).astype(np.float32)
            b = rng.uniform(1, 10, (2, k, m)).astype(np.float16).astype(np.float32)
            b[0, 0, 0] = NOT_HALF
            got = tng._run(torch, mm, ctx, "tf32", tng._dev(torch, "tf32", a), tng._dev(torch, "tf32", b), n, k, m,
                           flags=mm.FLAG_BATCH_SHARED_A, batch=2)
    for p, kind in enumerate(("no fit", "fit")):
        check(torch, mm, got[p], a[0], b[p], kind, p, n, k, m)


@pytest.mark.parametrize("kind", KINDS)
def test_host_chunks(torch, mm, monkeypatch, kind):
    """The host pipeline in 128-row chunks: the first pass runs on B, then per chunk of A; one second pass."""
    monkeypatch.setenv("MM_HOST_CHUNK_ROWS", "128")
    n = 1000                                         # 8 chunks, the last one short
    with mm.Context(0) as ctx:
        for seed in (40, 41):
            a, b = operands(kind, seed, n=n)
            got = ctx.gemm_host(mm.FLOAT, mm.MULTIPLY, mm.ADD, a, b, n, K, M)[0]
    check(torch, mm, got, a, b, kind, kind, n=n)


def test_multi_agreement_after_optimistic_pass(torch, mm):
    """mm_multi_execute on one device listed twice; only the second block's rows do not fit.  The first block's
    first pass finishes optimistically, the agreement clears its word afterwards, and its second pass writes TF32."""
    with mm.Multi(2, devices=[0, 0]) as multi:
        for seed in (50, 51):
            a, b = operands("late", seed)
            multi.upload(mm.FLOAT, a, b, N, K, M)
            multi.execute(mm.FLOAT, mm.MULTIPLY, mm.ADD, N, K, M)
            got = multi.download(mm.FLOAT, N, M)
    check(torch, mm, got, a, b, "late", "multi")
