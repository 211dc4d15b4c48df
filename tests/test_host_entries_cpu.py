"""The poisoning protocol of tests/host_poison.py against simulated host entries (no GPU needed).

`SimEntry` is a context of the host-pointer entries in numpy.  Its staged A, B, prepared B and C persist across
calls and are reallocated only to grow, as the library's ensure() does.  B arrives in 64-row slices, as in the
multi-GPU gather.  A is computed in row chunks, C in 128-column tiles, and C is copied out chunk by chunk.
Each defect below leaves one piece of that work undone, so the call returns what the staging held before:

* the last chunk's kernel is skipped;
* the last chunk's device-to-host copy is skipped;
* one slice of B is left out of the gather;
* the last column tile of C is never written;
* the prepared B of the previous call is reused;
* download serves a C that the last execute did not write.

The protocol rejects every defect and passes the correct entry.  The old check accepts every defect: it runs a call
that the defect does not touch, then the defective call on the same handle and data, and compares the bits.  The
defective call then returns the right answer from stale buffers, so even a comparison with the exact product passes.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import host_poison as hp  # noqa: E402

CHUNK_ROWS, TILE_COLS, SLICE_ROWS = 128, 128, 64
N, K, M = 300, 192, 272          # 3 row chunks (the last one short), 3 slices of B, 3 column tiles (the last one short)
DTYPES = [np.float32, np.uint8]
DEFECTS = ["skip_last_chunk_kernel", "skip_last_chunk_copy", "skip_b_slice", "skip_last_column_tile",
           "stale_prepared_b", "stale_download"]
LIFECYCLE_DEFECTS = {"stale_download"}


def product(dtype, a, b):
    """A B stored in dtype: float32 on small integers is exact; uint8 modulo 256."""
    if np.dtype(dtype).kind == "f":
        with np.errstate(invalid="ignore"):
            return (a.astype(np.float64) @ b.astype(np.float64)).astype(dtype)
    return ((a.astype(np.uint64) @ b.astype(np.uint64)) % 256).astype(dtype)


class SimEntry:
    """mm_gemm_host and the upload / execute / download lifecycle on one set of persistent staging arrays."""

    def __init__(self, dtype, defect=None):
        self.dtype = np.dtype(dtype)
        self.defect = defect
        self.staging = {}
        self.prepared_for = None
        self.resident = None

    def _buffer(self, name, size):
        buf = self.staging.get(name)
        if buf is None or buf.size < size:
            buf = self.staging[name] = np.zeros(size, self.dtype)
        return buf

    def _upload(self, a, b, n, k, m):
        sa, sb = self._buffer("a", n * k), self._buffer("b", k * m)
        self._buffer("c", n * m)
        sa[: n * k] = a
        for s0 in range(0, k, SLICE_ROWS):
            s1 = min(k, s0 + SLICE_ROWS)
            if self.defect == "skip_b_slice" and s1 == k and s0 > 0:
                continue
            sb[s0 * m: s1 * m] = b[s0 * m: s1 * m]
        if not (self.defect == "stale_prepared_b" and self.prepared_for == (k, m)):
            self._buffer("bt", k * m)[: k * m] = sb[: k * m].reshape(k, m).T.reshape(-1)
        self.prepared_for = (k, m)

    def _compute(self, n, k, m, chunk_rows, into):
        a = self.staging["a"][: n * k].reshape(n, k)
        bt = self.staging["bt"][: k * m].reshape(m, k)
        c = into[: n * m].reshape(n, m)
        starts = range(0, n, chunk_rows)
        for i, r0 in enumerate(starts):
            if self.defect == "skip_last_chunk_kernel" and i == len(starts) - 1:
                continue
            for c0 in range(0, m, TILE_COLS):
                if self.defect == "skip_last_column_tile" and c0 + TILE_COLS >= m:
                    continue
                c[r0: r0 + chunk_rows, c0: c0 + TILE_COLS] = product(self.dtype, a[r0: r0 + chunk_rows],
                                                                     bt[c0: c0 + TILE_COLS].T)

    def gemm_host(self, a, b, n, k, m, out, chunk_rows=CHUNK_ROWS):
        self._upload(a, b, n, k, m)
        self._compute(n, k, m, chunk_rows, self.staging["c"])
        c = self.staging["c"][: n * m].reshape(n, m)
        starts = range(0, n, chunk_rows)
        for i, r0 in enumerate(starts):
            if self.defect == "skip_last_chunk_copy" and i == len(starts) - 1:
                continue
            out[r0: r0 + chunk_rows] = c[r0: r0 + chunk_rows]
        return out

    def upload(self, a, b, n, k, m):
        self._upload(a, b, n, k, m)
        self.resident = (n, k, m)

    def execute(self):
        n, k, m = self.resident
        into = np.empty(n * m, self.dtype) if self.defect == "stale_download" else self.staging["c"]
        self._compute(n, k, m, n, into)

    def download(self, out):
        n, _, m = self.resident
        out[...] = self.staging["c"][: n * m].reshape(n, m)
        return out

    def lifecycle(self, a, b, n, k, m, out):
        self.upload(a, b, n, k, m)
        self.execute()
        return self.download(out)


def _data(dtype, seed=0):
    rng = np.random.default_rng(seed)
    if np.dtype(dtype).kind == "f":
        draw = lambda shape: (rng.integers(1, 9, size=shape) * rng.choice([-1, 1], size=shape)).astype(dtype)  # noqa: E731
    else:
        draw = lambda shape: rng.integers(0, 256, size=shape, dtype=np.uint8)  # noqa: E731
    a, b = draw((N, K)), draw((K, M))
    return a.reshape(-1), b.reshape(-1), product(dtype, a, b)


def _entry_call(entry, lifecycle, chunk_rows=CHUNK_ROWS):
    if lifecycle:
        return lambda a, b, out, poison: entry.lifecycle(a, b, N, K, M, out)
    return lambda a, b, out, poison: entry.gemm_host(a, b, N, K, M, out, chunk_rows=chunk_rows)


# ---- the protocol's own pieces --------------------------------------------------------------------------------------

def test_poison_bytes_are_nan_in_every_floating_type():
    for dt in (np.float16, np.float32, np.float64):
        assert np.isnan(hp.poison_c(dt, 2, 2, hp.FLOAT_ROUNDS[0])).all()
    assert hp.nan_mask(hp.poison_c(np.uint16, 2, 2, hp.FLOAT_ROUNDS[0]), bf16=True).all()
    assert hp.nan_mask(np.array([hp.BF16_NAN], np.uint16), bf16=True).all()


@pytest.mark.parametrize("dt", [np.int32, np.uint32, np.uint8])
def test_integer_rounds_differ_in_every_element(dt):
    (p1, q1, h1), (p2, q2, h2) = hp.INT_ROUNDS
    assert np.asarray(p1 * q1).astype(dt) != np.asarray(p2 * q2).astype(dt)
    assert h1 != h2
    for k in (64, 256, 33088):        # C = p q at any K: only row 0 of B is nonzero
        for p, q, h in hp.INT_ROUNDS:
            a, b = hp.poison_operands(dt, 3, k, 64, (p, q, h))
            c = (a.reshape(3, k).astype(np.uint64) @ b.reshape(k, 64).astype(np.uint64)).astype(dt)
            assert (c == np.asarray(p * q).astype(dt)).all()


def test_same_bits_treats_nan_payloads_as_equal_and_nothing_else():
    x = np.array([1.0, np.nan, -0.0], np.float32)
    y = np.array([1.0, np.float32(np.uint32(0x7FC00001).view(np.float32)), -0.0], np.float32)
    assert hp.same_bits(x, y)
    assert not hp.same_bits(x, np.array([1.0, np.nan, 0.0], np.float32))     # the sign of zero counts
    assert not hp.same_bits(x, np.array([1.0, 2.0, -0.0], np.float32))


# ---- simulated entries ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: np.dtype(d).name)
@pytest.mark.parametrize("how", ["one_chunk", "chunked", "lifecycle"])
def test_correct_entry_passes(dtype, how):
    a, b, want = _data(dtype)
    entry = SimEntry(dtype)
    call = _entry_call(entry, how == "lifecycle", chunk_rows=N if how == "one_chunk" else CHUNK_ROWS)
    hp.run(call, a, b, want, dtype, N, K, M)


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: np.dtype(d).name)
@pytest.mark.parametrize("defect", DEFECTS)
def test_protocol_rejects_each_defect(dtype, defect):
    a, b, want = _data(dtype)
    entry = SimEntry(dtype, defect)
    with pytest.raises(AssertionError):
        hp.run(_entry_call(entry, defect in LIFECYCLE_DEFECTS), a, b, want, dtype, N, K, M)


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: np.dtype(d).name)
@pytest.mark.parametrize("defect", DEFECTS)
def test_old_same_bits_check_accepts_each_defect(dtype, defect):
    """A correct call, then the defective one on the same handle, data and output buffer: same bits, and even equal
    to the exact product, because every skipped piece of work finds the right bytes already in place."""
    a, b, want = _data(dtype)
    entry = SimEntry(dtype)
    out = np.empty((N, M), dtype)
    first = entry.gemm_host(a, b, N, K, M, out, chunk_rows=N).copy()
    entry.defect = defect
    second = _entry_call(entry, defect in LIFECYCLE_DEFECTS)(a, b, out, False)
    assert hp.same_bits(second, first)
    assert hp.same_bits(second, want)
