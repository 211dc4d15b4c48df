"""mm_kernel_enqueue_witness on an H100 (run with `-m gpu`): C and the Min / Max witness W of every (type, Map, Min |
Max) on the data of tests/witness_data.py, against tests/witness_naive.py.

Shapes as the semiring coverage suite (semiring_data.gpu_shape: N = 259, M = 256 + BK, K = 10 k-tiles).  Matrix:
every pair under MM_FLAG_EXACT; float at flags = 0 (FMNMX); the 4-byte types with semiring_ring = 0 (the
register-staged witness kernel); every pair with MM_FLAG_TRANSPOSED_A; per type and reduce a batch of three problems
under each of the four MM_FLAG_BATCH_SHARED_* combinations.  Every call writes into C poisoned with 0xFF (and again
0x00 for integer types) and W poisoned with 0xA5 bytes (0xA5A5A5A5 is no valid k, 0xFF.. would read as NONE), each
followed by a 4 KiB guard that must stay as it was.  Checked per element: C has the bytes of mm_kernel_enqueue_batched
with the same arguments; W is witness_naive's exactly; and the invariant of include/mm_b200.h (C is term W, or the
identity where W is NONE).

Also: argument validation (one case per rule), a graph capture and replay, per-call profiling, and three 8192^3
products (float (Add, Min) at flags 0 and under EXACT, int32 (Add, Max)): C byte for byte against the plain call, the
invariant on every element on the device, W against the reference on sampled rows.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import full_size_check as fsc  # noqa: E402
import semiring_data as sd  # noqa: E402
import witness_data as wd  # noqa: E402
import witness_naive as wn  # noqa: E402
from semiring_data import ADD, FLOAT, FLOATING, INT32, MAX, MIN, UINT32  # noqa: E402

pytestmark = pytest.mark.gpu

TA, EXACT, SHARED_A, SHARED_B = 1, 2, 8, 16
SEED = 5
BATCH = 3
PAIRS = [(dt, mp, rd) for dt in sd.TYPES for mp in sd.OPS for rd in (MIN, MAX)]
DEFAULT = [(FLOAT, mp, rd, 0) for mp in sd.OPS for rd in (MIN, MAX)]
STAGED = [(dt, mp, rd, EXACT) for dt, mp, rd in PAIRS if dt in (FLOAT, INT32, UINT32)] + DEFAULT
BATCHED = [(dt, (rd + dt) % 5, rd, sh) for dt in sd.TYPES for rd in (MIN, MAX)
           for sh in (0, SHARED_A, SHARED_B, SHARED_A | SHARED_B)]
W_POISON = 0xA5


def _ids(cases):
    return ["%s-f%d" % (sd.pair_name(*c[:3]), c[3]) if len(c) > 3 else sd.pair_name(*c) for c in cases]


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


@pytest.fixture(scope="module")
def staged_ctx(mm):
    c = mm.Context(0)
    c.set_tuning(semiring_ring=0)
    yield c
    c.close()


_DATA, _WANT = {}, {}


def data(dt, mp, rd, seed):
    key = (dt, mp, rd, seed)
    if key not in _DATA:
        n, m, k = sd.gpu_shape(dt)
        _DATA[key] = wd.case(dt, mp, rd, n, k, m, seed)
    return _DATA[key]


def want(dt, mp, rd, fmnmx, a, b, key):
    if key not in _WANT:
        _WANT[key] = wn.witness(dt, mp, rd, a, b, fmnmx=fmnmx)
    return _WANT[key]


def _nan(x, dt):
    if dt == sd.BF16:
        return (x & 0x7FFF) > 0x7F80
    return np.isnan(x) if dt in FLOATING else np.zeros(x.shape, bool)


def check_invariant(what, dt, mp, rd, fmnmx, a, b, c, w):
    """C is term W (bits on the literal path, NaN payload free; the number under FMNMX), or the identity at NONE."""
    ar = sd._Arith(dt)
    av, bv = ar.load(a), ar.load(b)
    cv = ar.load(c)
    hit = w != wn.NONE
    assert (w[hit] < a.shape[1]).all(), "%s: witness out of range" % what
    ws = np.where(hit, w, 0).astype(np.int64)
    rows = np.arange(c.shape[0])[:, None]
    cols = np.arange(c.shape[1])[None, :]
    term = ar.store(wn._term(ar, mp, fmnmx, av[rows, ws], bv[ws, cols]))
    ident = np.full(c.shape, sd.identity(dt, rd), dtype=c.dtype)
    expect = np.where(hit, term, ident)
    if fmnmx:
        ok = (np.where(hit, ar.load(term), ar.load(ident)) == cv)
    else:   # the same bits, any NaN equal to any NaN
        nan_e, nan_c = _nan(expect, dt), _nan(c, dt)
        u = np.dtype("u%d" % sd.SIZE[dt])
        ok = (nan_e & nan_c) | (~nan_e & ~nan_c & (expect.view(u) == c.view(u)))
    if not ok.all():
        i, j = (int(v) for v in np.argwhere(~ok)[0])
        raise AssertionError("%s: %d elements break the invariant; first (%d, %d): C %r, W %d" % (
            what, int((~ok).sum()), i, j, c[i, j], w[i, j]))


def compare(what, got, exp, name):
    if not np.array_equal(got, exp):
        bad = np.argwhere(got != exp)
        i, j = (int(v) for v in bad[0])
        raise AssertionError("%s: %s differs at %d of %d elements; first (%d, %d): got %r, want %r" % (
            what, name, len(bad), got.size, i, j, got[i, j], exp[i, j]))


def run(torch, mm, c, dt, mp, rd, flags, seeds):
    """One witness call over len(seeds) problems (shared operands per the flags), checked against everything."""
    n, m, k = sd.gpu_shape(dt)
    batch = len(seeds)
    fmnmx = dt == FLOAT and not flags & EXACT
    probs = [data(dt, mp, rd, s) for s in seeds]
    a_of = [probs[0][0] if flags & SHARED_A else p[0] for p in probs]
    b_of = [probs[0][1] if flags & SHARED_B else p[1] for p in probs]
    a_up = a_of[:1] if flags & SHARED_A else a_of
    b_up = b_of[:1] if flags & SHARED_B else b_of
    a_host = [np.ascontiguousarray(x.T) if flags & TA else x for x in a_up]
    da = torch.from_numpy(np.concatenate([x.reshape(-1) for x in a_host]).view(np.uint8).copy()).cuda()
    db = torch.from_numpy(np.concatenate([x.reshape(-1) for x in b_up]).view(np.uint8).copy()).cuda()
    what = "%s flags %d batch %d" % (sd.pair_name(dt, mp, rd), flags, batch)
    cbytes, wbytes = batch * n * m * sd.SIZE[dt], batch * n * m * 4
    plain = torch.zeros(cbytes, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    torch.cuda.synchronize()
    c.enqueue_batched(dt, mp, rd, da.data_ptr(), db.data_ptr(), plain.data_ptr(), n, k, m, batch, flags=flags,
                      stream=stream)
    torch.cuda.synchronize()
    plain = plain.cpu().numpy()
    for poison in ((0xFF,) if dt in FLOATING else (0xFF, 0x00)):
        craw = torch.full((cbytes + fsc.GUARD,), poison, dtype=torch.uint8, device="cuda")
        wraw = torch.full((wbytes + fsc.GUARD,), W_POISON, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        c.enqueue_witness(dt, mp, rd, da.data_ptr(), db.data_ptr(), craw.data_ptr(), wraw.data_ptr(), n, k, m,
                          batch=batch, flags=flags, stream=stream)
        torch.cuda.synchronize()
        fsc.check_guard(torch, what + " (C)", craw[cbytes:], poison)
        fsc.check_guard(torch, what + " (W)", wraw[wbytes:], W_POISON)
        cgot = craw[:cbytes].cpu().numpy()
        compare(what, cgot.reshape(batch, -1), plain.reshape(batch, -1), "C against mm_kernel_enqueue_batched")
        wgot = wraw[:wbytes].cpu().numpy().view(np.uint32).reshape(batch, n, m)
        cval = cgot.view(sd.NP[dt]).reshape(batch, n, m)
        for z in range(batch):
            key = (dt, mp, rd, fmnmx, seeds[0 if flags & SHARED_A else z], seeds[0 if flags & SHARED_B else z])
            _, wexp = want(dt, mp, rd, fmnmx, a_of[z], b_of[z], key)
            compare("%s problem %d" % (what, z), wgot[z], wexp, "W")
            check_invariant("%s problem %d" % (what, z), dt, mp, rd, fmnmx, a_of[z], b_of[z], cval[z], wgot[z])


@pytest.mark.parametrize("dt,mp,rd", PAIRS, ids=_ids(PAIRS))
def test_every_pair_exact(torch, mm, ctx, dt, mp, rd):
    run(torch, mm, ctx, dt, mp, rd, EXACT, [SEED])


@pytest.mark.parametrize("dt,mp,rd,flags", DEFAULT, ids=_ids(DEFAULT))
def test_float_default_flags(torch, mm, ctx, dt, mp, rd, flags):
    run(torch, mm, ctx, dt, mp, rd, flags, [SEED])


@pytest.mark.parametrize("dt,mp,rd,flags", STAGED, ids=_ids(STAGED))
def test_register_staged_kernel(torch, mm, staged_ctx, dt, mp, rd, flags):
    run(torch, mm, staged_ctx, dt, mp, rd, flags, [SEED])


@pytest.mark.parametrize("dt,mp,rd", PAIRS, ids=_ids(PAIRS))
def test_transposed_a(torch, mm, ctx, dt, mp, rd):
    run(torch, mm, ctx, dt, mp, rd, EXACT | TA, [SEED])


@pytest.mark.parametrize("dt,mp,rd,flags", BATCHED, ids=_ids(BATCHED))
def test_batch_of_three(torch, mm, ctx, dt, mp, rd, flags):
    run(torch, mm, ctx, dt, mp, rd, EXACT | flags, [SEED + z for z in range(BATCH)])


def test_argument_validation(torch, mm, ctx):
    n, k, m = 128, 64, 128
    a = torch.zeros(n * k, dtype=torch.float32, device="cuda")
    b = torch.zeros(k * m, dtype=torch.float32, device="cuda")
    c = torch.zeros(n * m, dtype=torch.float32, device="cuda")
    w = torch.zeros(n * m + 4, dtype=torch.int32, device="cuda")
    p = (a.data_ptr(), b.data_ptr(), c.data_ptr())
    torch.cuda.synchronize()
    ctx.enqueue_witness(FLOAT, ADD, MIN, *p, w.data_ptr(), n, k, m)   # the valid call
    torch.cuda.synchronize()
    cases = {
        "null W": ((FLOAT, ADD, MIN) + p + (None, n, k, m), {}),
        "W not 16-byte aligned": ((FLOAT, ADD, MIN) + p + (w.data_ptr() + 4, n, k, m), {}),
        "Add reduce": ((FLOAT, ADD, ADD) + p + (w.data_ptr(), n, k, m), {}),
        "And reduce": ((FLOAT, ADD, sd.AND) + p + (w.data_ptr(), n, k, m), {}),
        "Multiply reduce": ((FLOAT, ADD, sd.MULTIPLY) + p + (w.data_ptr(), n, k, m), {}),
        "batch 0": ((FLOAT, ADD, MIN) + p + (w.data_ptr(), n, k, m), {"batch": 0}),
        "null C": ((FLOAT, ADD, MIN, a.data_ptr(), b.data_ptr(), None, w.data_ptr(), n, k, m), {}),
        "unknown type": ((99, ADD, MIN) + p + (w.data_ptr(), n, k, m), {}),
    }
    for name, (args, kw) in cases.items():
        with pytest.raises(mm.MMError) as e:
            ctx.enqueue_witness(*args, **kw)
        assert e.value.code == 1, name
    with pytest.raises(mm.MMError) as e:   # K not a multiple of the memory width
        ctx.enqueue_witness(FLOAT, ADD, MIN, *p, w.data_ptr(), n, 24, m)
    assert e.value.code == 2
    with pytest.raises(mm.MMError) as e:
        ctx.enqueue_witness(FLOAT, ADD, MIN, *p, w.data_ptr(), n, k, m, batch=65536)
    assert e.value.code == 5


def test_graph_capture_and_profiling(torch, mm):
    dt, mp, rd = FLOAT, ADD, MIN
    n, m, k = sd.gpu_shape(dt)
    a, b = data(dt, mp, rd, SEED)
    da, db = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    c0, w0 = torch.empty((n, m), device="cuda"), torch.empty((n, m), dtype=torch.int32, device="cuda")
    c1, w1 = torch.full_like(c0, -1.0), torch.full_like(w0, -1)
    torch.cuda.synchronize()
    with mm.Context(0) as ctx:
        ctx.enqueue_witness(dt, mp, rd, da.data_ptr(), db.data_ptr(), c0.data_ptr(), w0.data_ptr(), n, k, m,
                            stream=torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):   # a fresh context: no reserve, the call needs no scratch
            ctx.enqueue_witness(dt, mp, rd, da.data_ptr(), db.data_ptr(), c1.data_ptr(), w1.data_ptr(), n, k, m,
                                stream=s.cuda_stream)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(c0.view(torch.int32), c1.view(torch.int32)) and torch.equal(w0, w1)
        del g
        ctx.set_profiling(True)
        ctx.enqueue_witness(dt, mp, rd, da.data_ptr(), db.data_ptr(), c1.data_ptr(), w1.data_ptr(), n, k, m)
        prep, main, calls = ctx.profile_read()
        assert calls == 1 and main > 0 and prep < main
    _, wexp = wn.witness(dt, mp, rd, a, b, fmnmx=True)
    assert np.array_equal(w0.cpu().numpy().view(np.uint32), wexp)


FULL = [(FLOAT, ADD, MIN, 0), (FLOAT, ADD, MIN, EXACT), (INT32, ADD, MAX, 0)]


@pytest.mark.parametrize("dt,mp,rd,flags", FULL, ids=_ids(FULL))
def test_full_size(torch, mm, ctx, dt, mp, rd, flags):
    """8192^3: C byte for byte against the plain call; on every element, C is term W computed on the device; W
    against the reference on sampled rows."""
    n = k = m = 8192
    gen = torch.Generator(device="cuda")
    gen.manual_seed(11)
    if dt == FLOAT:   # U[1, 10] rounded to 1/16: exact ties between terms are common
        a = (torch.randint(16, 160, (n, k), generator=gen, device="cuda") / 16.0).float()
        b = (torch.randint(16, 160, (k, m), generator=gen, device="cuda") / 16.0).float()
    else:
        a = torch.randint(-2 ** 20, 2 ** 20, (n, k), generator=gen, device="cuda", dtype=torch.int32)
        b = torch.randint(-2 ** 20, 2 ** 20, (k, m), generator=gen, device="cuda", dtype=torch.int32)
    c_plain = torch.zeros((n, m), dtype=a.dtype, device="cuda")
    c = torch.full((n, m), -1, dtype=a.dtype, device="cuda")
    w = torch.full((n, m), -0x5A5A5A5B, dtype=torch.int32, device="cuda")   # 0xA5A5A5A5
    s = torch.cuda.current_stream().cuda_stream
    torch.cuda.synchronize()   # the operands and poisoned buffers are written before the library's stream reads them
    ctx.enqueue(dt, mp, rd, a.data_ptr(), b.data_ptr(), c_plain.data_ptr(), n, k, m, flags=flags, stream=s)
    ctx.enqueue_witness(dt, mp, rd, a.data_ptr(), b.data_ptr(), c.data_ptr(), w.data_ptr(), n, k, m, flags=flags,
                        stream=s)
    torch.cuda.synchronize()
    what = "%s flags %d 8192^3" % (sd.pair_name(dt, mp, rd), flags)
    diff = c.view(torch.int32) != c_plain.view(torch.int32)
    if bool(diff.any()):
        i, j = (int(v) for v in diff.nonzero()[0])
        terms = a[i] + b[:, j]
        best = terms.min() if rd == MIN else terms.max()
        raise AssertionError("%s: C differs from the plain call at %d elements; first (%d, %d): witness call %r, "
                             "plain call %r, Naive<> %r" % (what, int(diff.sum()), i, j, c[i, j].item(),
                                                            c_plain[i, j].item(), best.item()))
    assert bool(((w >= 0) & (w < k)).all()), what + ": a witness outside [0, K)"   # every term beats the identity
    for r0 in range(0, n, 2048):   # C[i, j] == a[i, W] + b[W, j], in row blocks
        wl = w[r0:r0 + 2048].long()
        term =a[r0:r0 + 2048].gather(1, wl) + b[wl, torch.arange(m, device="cuda")[None, :]]
        ok = term.view(torch.int32) == c[r0:r0 + 2048].view(torch.int32)
        assert bool(ok.all()), "%s: %d elements of rows %d.. are not term W" % (what, int((~ok).sum()), r0)
    rows = [0, 1, 4095, 8191]
    _, wexp = wn.witness(dt, mp, rd, a[rows].cpu().numpy(), b.cpu().numpy(), fmnmx=dt == FLOAT and not flags & EXACT)
    assert np.array_equal(w[rows].cpu().numpy().view(np.uint32), wexp), what + ": W differs on the sampled rows"
