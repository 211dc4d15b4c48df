"""Test infrastructure: the poisoning protocol of the host-pointer entries.

mm_gemm_host, mm_multi_gemm_host and the mm_multi upload / execute / download lifecycle keep A, B and C in
per-context device buffers that later calls reuse, and the tensor-core path keeps the prepared B in the context's
scratch.  A call that skips a chunk's kernel or copy, a slice of B's gather or a column tile of C hands back what
those buffers held.  That is usually the previous call's bytes, which are the right answer whenever a test repeats
a call on the same data, so comparing a call with an earlier one cannot see the defect.

The protocol makes every stale byte wrong.  Before the call under test, a poison call through the same handle, with
the same type, flags and shape, leaves poison in the staged A, B, prepared B and C:

* floating types: all-NaN A and B in (Multiply, Add); NaN reaches C on every path;
* integer types: A = p everywhere, B = q in row 0 and 0 elsewhere, so that C = p * q exactly at any K.  Each case
  runs twice, with two (p, q) whose C differ: an element that was never written fails at least one of the runs.

The host C the call writes into is prefilled with poison bytes too (0xFF is NaN in every floating type; the two
integer runs use two different bytes).  The expected C must come from arithmetic that shares nothing with the
entry's earlier output, and for floating types it must be NaN-free, so that the poison cannot pass for a result.

tests/test_host_entries_gpu.py runs the protocol on the library's entries; tests/test_host_entries_cpu.py shows on
simulated entries that it rejects each stale-data defect that the old "same bits as the previous call" check accepts.
bfloat16 values are np.uint16 bit patterns (`bf16=True`).
"""
import numpy as np

BF16_NAN = 0x7FC0
# (p, q, host C byte) of the two integer runs: C = 90 and 117 in every integer type
INT_ROUNDS = ((1, 0x5A, 0x5A), (3, 0x27, 0xA5))
FLOAT_ROUNDS = ((None, None, 0xFF),)


def is_float(dtype, bf16=False):
    return bf16 or np.dtype(dtype).kind == "f"


def rounds(dtype, bf16=False):
    return FLOAT_ROUNDS if is_float(dtype, bf16) else INT_ROUNDS


def nan_mask(x, bf16=False):
    x = np.asarray(x)
    if bf16:
        return (x.astype(np.uint16) & 0x7FFF) > 0x7F80
    if x.dtype.kind == "f":
        return np.isnan(x)
    return np.zeros(x.shape, dtype=bool)


def poison_operands(dtype, n, k, m, rnd, bf16=False):
    """Flat A (n * k elements, either layout) and B (k * m, row-major) of one poison call."""
    p, q, _ = rnd
    if is_float(dtype, bf16):
        nan = BF16_NAN if bf16 else np.nan
        return np.full(n * k, nan, dtype=dtype), np.full(k * m, nan, dtype=dtype)
    a = np.full(n * k, p, dtype=dtype)
    b = np.zeros(k * m, dtype=dtype)
    b[:m] = q
    return a, b


def poison_c(dtype, n, m, rnd):
    """An n x m host C whose every byte is the run's poison byte."""
    return np.full(n * m * np.dtype(dtype).itemsize, rnd[2], dtype=np.uint8).view(dtype).reshape(n, m)


def same_bits(got, want, bf16=False):
    """Bit equality, except that any NaN equals any NaN (payloads are free)."""
    got, want = np.asarray(got).reshape(-1), np.asarray(want).reshape(-1)
    if got.dtype != want.dtype or got.shape != want.shape:
        return False
    ng, nw = nan_mask(got, bf16), nan_mask(want, bf16)
    if not np.array_equal(ng, nw):
        return False
    u = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[got.dtype.itemsize]
    return bool(np.array_equal(got.view(u)[~ng], want.view(u)[~nw]))


def assert_same_bits(got, want, bf16=False):
    if not same_bits(got, want, bf16):
        g, w = np.asarray(got).reshape(-1), np.asarray(want).reshape(-1)
        u = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[g.dtype.itemsize]
        bad = np.flatnonzero((g.view(u) != w.view(u)) & ~(nan_mask(g, bf16) & nan_mask(w, bf16)))
        raise AssertionError("%d of %d elements differ; first at flat %d: got %r want %r" % (
            bad.size, g.size, bad[0], g[bad[0]], w[bad[0]]))


def run(call, a, b, want, dtype, n, k, m, bf16=False, compare=None):
    """The protocol around one entry.  `call(a, b, out, poison)` runs the entry on flat host operands a, b and writes
    C into `out` (returning it); poison=True marks the poison call, which the caller runs in (Multiply, Add) with the
    flags of the call under test.  `compare(got, want)` asserts (default: bit equality, NaN payloads free)."""
    compare = compare or (lambda g, w: assert_same_bits(g, w, bf16))
    if is_float(dtype, bf16):
        assert not nan_mask(want, bf16).any(), "the expected C holds NaN: the poison would be invisible"
    for rnd in rounds(dtype, bf16):
        pa, pb = poison_operands(dtype, n, k, m, rnd, bf16)
        poisoned = np.asarray(call(pa, pb, poison_c(dtype, n, m, rnd), True))
        if is_float(dtype, bf16):
            assert nan_mask(poisoned, bf16).all(), "the poison call left non-NaN elements in C"
        else:
            assert (poisoned == np.asarray(rnd[0] * rnd[1]).astype(dtype)).all(), "the poison call's C is not p * q"
        out = poison_c(dtype, n, m, rnd)
        got = call(a, b, out, False)
        assert got is out or np.shares_memory(got, out), "the entry did not write into the caller's C"
        compare(np.asarray(out).reshape(n, m), np.asarray(want).reshape(n, m))
