"""Every CUDA-core semiring kernel at multi-tile shapes, on data that shows each k-tile, seed and rounding (run with
`-m gpu` on an H100).

Shape per type (BK = 64 bytes of K): N = 259 (three 128-row tiles, the last of 3 rows), M = 256 + BK (three 128-column
tiles, the last partial), K = 10 BK.  The ring kernel's 4 stages wrap more than twice, so both phases of every full and
empty barrier are used; the register-staged kernel's two B buffers alternate five times.

Matrix: every (type, Map, Reduce) under MM_FLAG_EXACT; flags = 0 for float pairs with Min or Max (FMNMX); float, int32
and uint32 also with semiring_ring = 0 (the register-staged kernel); every pair with MM_FLAG_TRANSPOSED_A (always the
register-staged kernel; N = 259 is not a multiple of the vector width); and per type and reduce one batch of three
problems with their own data through mm_kernel_enqueue_batched (blockIdx.z and the per-problem offsets).

Data: tests/semiring_data.py, whose power tests/test_semiring_data_cpu.py shows without a GPU.  Every call goes through
Context.enqueue (or enqueue_batched) into a C of 0xFF bytes followed by a 4 KiB guard; integer types run again with
0x00, since 0xFF is a legitimate uint8_t result.  The reference is Naive<> on the CPU (the oracle; tests/bf16_naive.py
for bfloat16), compared bit for bit, any NaN equal to any NaN.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import full_size_check as fsc  # noqa: E402
import semiring_data as sd  # noqa: E402
from semiring_data import BF16, FLOAT, FLOATING, INT32, MAX, MIN, UINT32  # noqa: E402

pytestmark = pytest.mark.gpu

TA, EXACT = 1, 2
SEED = 5
PAIRS = [(dt, mp, rd) for dt in sd.TYPES for mp in sd.OPS for rd in sd.OPS]
FMNMX = [(FLOAT, mp, rd) for mp in sd.OPS for rd in sd.OPS if {mp, rd} & {MIN, MAX}]
STAGED = [p + (EXACT,) for p in PAIRS if p[0] in (FLOAT, INT32, UINT32)] + [p + (0,) for p in FMNMX]
BATCHED = [(dt, (rd + dt) % 5, rd) for dt in sd.TYPES for rd in sd.OPS]   # every Map appears under every reduce
BATCH = 3


def _ids(cases):
    return [sd.pair_name(*c[:3]) + ("" if len(c) < 4 or c[3] & EXACT else "-fmnmx") for c in cases]


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
    """A context whose 4-byte semirings take the register-staged kernel instead of the TMA ring."""
    c = mm.Context(0)
    c.set_tuning(semiring_ring=0)
    yield c
    c.close()


_CASES = {}


def case(oracle, dt, mp, rd, exact=True, seed=SEED):
    """(A, B, Naive<> C) at the type's shape."""
    key = (dt, mp, rd, exact, seed)
    if key not in _CASES:
        n, m, k = sd.gpu_shape(dt)
        a, b = sd.discriminating(dt, mp, rd, n, k, m, seed, exact)
        _CASES[key] = (a, b, sd.reference(oracle, dt, mp, rd, a, b, n, k, m))
    return _CASES[key]


def _nan(x, dt):
    if dt == BF16:
        return (x & 0x7FFF) > 0x7F80
    return np.isnan(x) if dt in FLOATING else np.zeros(x.shape, bool)


def compare(what, dt, got, want, poison, z=0, batch=1):
    """Every element, bit for bit (any NaN equals any NaN); the report names (row, col), the CTA and the k-tiles."""
    w = np.dtype("u%d" % sd.SIZE[dt])
    gn, wn = _nan(got, dt), _nan(want, dt)
    wrong = (gn != wn) | (~gn & ~wn & (got.view(w) != want.view(w)))
    if wrong.any():
        row, col = (int(v) for v in np.argwhere(wrong)[0])
        n, m = got.shape
        k = sd.gpu_shape(dt)[2]
        held = int((got.view(np.uint8).reshape(n, m, -1) == poison).all(axis=2)[wrong].sum())
        raise AssertionError(
            "%s: %d of %d elements wrong (%d still hold the poison byte 0x%02X); first at (row %d, col %d): got %r, "
            "want %r; CTA blockIdx (x %d, y %d, z %d) of a %d x %d x %d grid, %d k-tiles of %d" % (
                what, int(wrong.sum()), wrong.size, held, poison, row, col, got[row, col], want[row, col],
                col // sd.TILE, row // sd.TILE, z, -(-m // sd.TILE), -(-n // sd.TILE), batch,
                k // sd.bk(dt), sd.bk(dt)))


def run(torch, mm, c, dt, mp, rd, flags, problems):
    """C of each (A, B, want) problem through one enqueue (one problem) or one enqueue_batched (several)."""
    n, m, k = sd.gpu_shape(dt)
    assert mm.kernel_path(dt, mp, rd, flags) == "semiring_simt"
    what = "%s flags %d%s" % (sd.pair_name(dt, mp, rd), flags, " batch %d" % len(problems) if len(problems) > 1 else "")
    a_in = [np.ascontiguousarray(a.T) if flags & TA else a for a, _, _ in problems]
    da = torch.from_numpy(np.concatenate([x.reshape(-1) for x in a_in]).view(np.uint8).copy()).cuda()
    db = torch.from_numpy(np.concatenate([b.reshape(-1) for _, b, _ in problems]).view(np.uint8).copy()).cuda()
    nbytes = len(problems) * n * m * sd.SIZE[dt]
    for poison in ((0xFF,) if dt in FLOATING else (0xFF, 0x00)):
        raw = torch.full((nbytes + fsc.GUARD,), poison, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        stream = torch.cuda.current_stream().cuda_stream
        if len(problems) == 1:
            c.enqueue(dt, mp, rd, da.data_ptr(), db.data_ptr(), raw.data_ptr(), n, k, m, flags=flags, stream=stream)
        else:
            c.enqueue_batched(dt, mp, rd, da.data_ptr(), db.data_ptr(), raw.data_ptr(), n, k, m, len(problems),
                              flags=flags, stream=stream)
        torch.cuda.synchronize()
        fsc.check_guard(torch, what, raw[nbytes:], poison)
        got = raw[:nbytes].cpu().numpy().view(sd.NP[dt]).reshape(len(problems), n, m)
        for z, (_, _, want) in enumerate(problems):
            compare(what, dt, got[z], want, poison, z, len(problems))


@pytest.mark.parametrize("dt,mp,rd", PAIRS, ids=_ids(PAIRS))
def test_every_pair_exact(torch, mm, oracle, ctx, dt, mp, rd):
    run(torch, mm, ctx, dt, mp, rd, EXACT, [case(oracle, dt, mp, rd)])


@pytest.mark.parametrize("dt,mp,rd", FMNMX, ids=_ids(FMNMX))
def test_float_min_max_default_flags(torch, mm, oracle, ctx, dt, mp, rd):
    """flags = 0: FMNMX, on data without NaN, -0 or infinities, where it equals `(a < b) ? a : b`."""
    run(torch, mm, ctx, dt, mp, rd, 0, [case(oracle, dt, mp, rd, exact=False)])


@pytest.mark.parametrize("dt,mp,rd,flags", STAGED, ids=_ids(STAGED))
def test_register_staged_kernel(torch, mm, oracle, staged_ctx, dt, mp, rd, flags):
    run(torch, mm, staged_ctx, dt, mp, rd, flags, [case(oracle, dt, mp, rd, exact=bool(flags & EXACT))])


@pytest.mark.parametrize("dt,mp,rd", PAIRS, ids=_ids(PAIRS))
def test_transposed_a(torch, mm, oracle, ctx, dt, mp, rd):
    run(torch, mm, ctx, dt, mp, rd, EXACT | TA, [case(oracle, dt, mp, rd)])


@pytest.mark.parametrize("dt,mp,rd", BATCHED, ids=_ids(BATCHED))
def test_batch_of_three(torch, mm, oracle, ctx, dt, mp, rd):
    run(torch, mm, ctx, dt, mp, rd, EXACT, [case(oracle, dt, mp, rd, seed=SEED + z) for z in range(BATCH)])

