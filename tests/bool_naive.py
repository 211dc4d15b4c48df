"""Restatement of the bit-packed Boolean entries (include/mm_b200.h): mm_kernel_enqueue_bool and
mm_kernel_enqueue_bool_closure, in numpy, plus the test graphs and the plausible bugs the GPU data must reject.

Layout: element (i, j) of an R x L matrix is bit j % 8 (least significant first) of byte i*L/8 + j/8, which is
numpy.packbits(X, axis=-1, bitorder='little').  The product is the float32 matmul of 0/1 matrices followed by > 0,
exact while K < 2^24.  The closure is repeated squaring, R <- R | R.R, to a fixed point: paths of one or more edges.
"""
import numpy as np

B = 256  # the closure's block of indices (DESIGN.md 3.10); the result does not depend on it


def pack(x, bitorder="little"):
    return np.packbits(np.asarray(x, dtype=bool), axis=-1, bitorder=bitorder)


def unpack(p, cols, bitorder="little"):
    return np.unpackbits(np.asarray(p, dtype=np.uint8), axis=-1, count=cols, bitorder=bitorder)


def product(a, b):
    """0/1 arrays (..., N, K) and (..., K, M) -> (..., N, M) uint8."""
    return (np.matmul(a.astype(np.float32), b.astype(np.float32)) > 0).astype(np.uint8)


def closure(d):
    """Transitive closure of 0/1 arrays (..., N, N) by repeated squaring to a fixed point."""
    r = np.asarray(d, dtype=np.uint8).copy()
    while True:
        nxt = r | product(r, r)
        if np.array_equal(nxt, r):
            return r
        r = nxt


def closure_blocked(d, b=B, skip_round=None, skip_panels=False):
    """Blocked Floyd-Warshall on one 0/1 N x N array as the kernels run it, with optional faults: round `skip_round`
    left out, or phase 2 (the panels) left out of every round."""
    d = np.asarray(d, dtype=np.uint8).copy()
    n = d.shape[0]
    for r in range(0, (n + b - 1) // b):
        if r == skip_round:
            continue
        k = np.arange(r * b, min((r + 1) * b, n))
        o = np.setdiff1d(np.arange(n), k)
        blk = d[np.ix_(k, k)]
        for t in range(len(k)):  # Warshall: step t over the whole block at once equals the sequential step
            blk |= blk[:, t:t + 1] & blk[t:t + 1, :]
        d[np.ix_(k, k)] = blk
        if not skip_panels:
            d[np.ix_(k, o)] |= product(blk, d[np.ix_(k, o)])
            d[np.ix_(o, k)] |= product(d[np.ix_(o, k)], blk)
        d[np.ix_(o, o)] |= product(d[np.ix_(o, k)], d[np.ix_(k, o)])
    return d


# ---- test data --------------------------------------------------------------------------------------------------
def random_bits(shape, density, seed):
    """0/1 uint8 with each element 1 with probability `density` (1.0: all ones, 0.0: all zeros)."""
    rng = np.random.default_rng(seed)
    return (rng.random(shape) < density).astype(np.uint8)


def hamiltonian_cycle(n, seed):
    """One directed cycle through every vertex in random order: it crosses every block of indices, so every round of
    the blocked closure matters; the closure is all ones."""
    p = np.random.default_rng(seed).permutation(n)
    d = np.zeros((n, n), np.uint8)
    d[p, np.roll(p, -1)] = 1
    return d


def reversed_path(n):
    """n-1 -> n-2 -> ... -> 0: every edge runs against the index order of the blocks."""
    d = np.zeros((n, n), np.uint8)
    d[np.arange(1, n), np.arange(n - 1)] = 1
    return d


def random_dag(n, density, seed):
    """Edges from a random order's earlier to later vertices: the closure's diagonal stays 0."""
    rng = np.random.default_rng(seed)
    p = rng.permutation(n)
    upper = np.triu(rng.random((n, n)) < density, 1).astype(np.uint8)
    d = np.zeros((n, n), np.uint8)
    d[np.ix_(p, p)] = upper
    return d


# (n, k, m, density, seed) of the GPU product tests: counts from one to K (all ones) and all zeros
PRODUCT_CASES = [
    (1, 128, 128, 0.5, 1), (127, 384, 640, 0.01, 2), (129, 1152, 384, 0.001, 3), (1000, 16384, 128, 0.0005, 4),
    (1000, 1152, 640, 1.0, 5), (129, 384, 384, 0.0, 6), (1000, 384, 640, 0.2, 7), (127, 16384, 384, 0.002, 8),
    (1, 1152, 640, 0.05, 9), (129, 128, 128, 0.3, 10),
]


def product_operands(n, k, m, density, seed):
    return random_bits((n, k), density, seed), random_bits((k, m), density, seed + 1000)


# ---- plausible bugs ---------------------------------------------------------------------------------------------
def product_msb_first(a, b):
    """The product of a kernel that reads and writes bits most significant first, seen through the true layout."""
    k, m = a.shape[-1], b.shape[-1]
    a2, b2 = unpack(pack(a), k, "big"), unpack(pack(b), m, "big")
    return unpack(pack(product(a2, b2), "big"), m)


def product_dropped_k(a, b, drop_from):
    """K truncated at `drop_from` (a lost last 128-bit chunk or last 1,024-bit stage)."""
    return product(a[..., :drop_from], b[..., :drop_from, :])
