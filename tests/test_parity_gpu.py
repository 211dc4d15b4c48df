"""GPU parity tests (run with `-m gpu` on an H100): the CUDA hot path, called THROUGH THE C-ABI
(libmm_b200.so via ctypes), against the oracle on the same seeded inputs.

Bars (north_star / reference test/TestSimulation.cpp:75-92):
  * CUDA-core semiring path (any non-(Multiply,Add) semiring, every integer type, and every type
    under MM_FLAG_EXACT): BIT-EXACT against Naive<>.
  * tensor-core paths: the reference's own criterion |test-ref|/ref <= 1e-3, plus the tighter
    tolerances written below (measured headroom recorded in DESIGN.md):
        float  via tf32 wgmma (inputs rounded to nearest TF32): max rel err <= 5e-4
               (worst-case bound 2 * 2^-11 = 9.8e-4 for all-positive data, independent of K; the
               error averages down with K: 2.1e-4 observed at K = 48, 1e-4 at K = 1024)
        double via DMMA                                                : max rel err <= 1e-12
        half   via f16 wgmma (FP32 accumulate, one rounding to half at the end), against
               an FP64 evaluation of the same half inputs              : max rel err <= 1e-3
"""
import hashlib
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "golden.json")))

TOL = {"wgmma_tf32": 5e-4, "dmma_f64": 1e-12, "wgmma_f16": 1e-3}


def run_case(mm, oracle, dtype, mp, rd, n, k, m, flags=0, seed=5, scale=None):
    a, b = oracle.fill(dtype, n, k, m, seed)
    if scale is not None:
        a = (a.astype(np.float64) * scale).astype(a.dtype)
    ta = bool(flags & mm.FLAG_TRANSPOSED_A)
    c = mm.matrix_multiplication_kernel(a, b, n, k, m, dtype=dtype, map_op=mp, reduce_op=rd, flags=flags)
    ref = oracle.naive(dtype, mp, rd, a, b, n, k, m, transposed_a=ta, threads=8)
    return a, b, c, ref


def max_rel(c, ref):
    c64, r64 = c.astype(np.float64), ref.astype(np.float64)
    return float(np.max(np.abs(c64 - r64) / np.abs(r64)))


def _id(rec):
    return "%s-%dx%dx%d" % (rec["config"], rec["n"], rec["k"], rec["m"])


# ---------------------------------------------------------------------------------------------
# 1. golden vectors from the reference's Naive<> (tests/golden/golden.json)
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rec", GOLDEN, ids=_id)
def test_golden_vectors(mm, oracle, rec):
    dtype, mp, rd = rec["dtype"], rec["map"], rec["reduce"]
    n, k, m = rec["n"], rec["k"], rec["m"]
    flags = mm.FLAG_TRANSPOSED_A if rec["transposed_a"] else 0
    a, b = oracle.fill(dtype, n, k, m, rec["seed"])
    assert hashlib.sha256(a.tobytes()).hexdigest() == rec["a_sha256"]
    path = mm.kernel_path(dtype, mp, rd, flags)
    c = mm.matrix_multiplication_kernel(a, b, n, k, m, dtype=dtype, map_op=mp, reduce_op=rd, flags=flags)
    if path in ("semiring_simt", "wgmma_i8"):   # CUDA cores, and exact integer tensor cores: bit for bit
        assert hashlib.sha256(c.tobytes()).hexdigest() == rec["c_sha256"], "not bit-exact vs reference Naive<>"
    else:
        c64 = c.astype(np.float64)
        if dtype == mm.HALF:
            # the golden record accumulates in half (SURVEY.md trap 5): compare loosely here, the
            # tight half check is test_half_tensor_path_vs_fp64
            assert abs(c64.flat[0] - float(rec["c_first"])) / float(rec["c_first"]) < 2e-2
        else:
            assert abs(c64.flat[0] - float(rec["c_first"])) / float(rec["c_first"]) < TOL[path]
            assert abs(c64.flat[-1] - float(rec["c_last"])) / float(rec["c_last"]) < TOL[path]
            assert abs(c64.sum() - float(rec["c_sum"])) / float(rec["c_sum"]) < TOL[path]
    # the exact path must reproduce the record bit for bit for every configuration
    ce = mm.matrix_multiplication_kernel(a, b, n, k, m, dtype=dtype, map_op=mp, reduce_op=rd,
                                         flags=flags | mm.FLAG_EXACT)
    assert hashlib.sha256(ce.tobytes()).hexdigest() == rec["c_sha256"]


# ---------------------------------------------------------------------------------------------
# 2. tensor-core paths vs the oracle: reference criterion + stated tolerance
# ---------------------------------------------------------------------------------------------
TENSOR_SHAPES = [
    (256, 256, 256),     # BASELINE config 1
    (513, 528, 528),     # the reference's CTest shape (CMakeLists.txt:155-159): ragged N, K % 32 != 0
    (1, 16, 16),         # smallest legal float shape
    (128, 2048, 256),    # exactly one tile, long K
    (129, 48, 272),      # one row past a tile, K tail of 16, M tail of 16
    (1024, 1024, 1024),
]


@pytest.mark.parametrize("n,k,m", TENSOR_SHAPES)
def test_float_tensor_path(mm, oracle, n, k, m):
    a, b, c, ref = run_case(mm, oracle, mm.FLOAT, mm.MULTIPLY, mm.ADD, n, k, m)
    assert oracle.verify(oracle.FLOAT, c, ref) == -1          # the reference's own 1e-3 check
    assert max_rel(c, ref) <= TOL["wgmma_tf32"]


@pytest.mark.parametrize("n,k,m", [(256, 256, 256), (513, 528, 528), (1, 8, 8), (130, 24, 136), (1024, 1024, 1024)])
def test_double_tensor_path(mm, oracle, n, k, m):
    a, b, c, ref = run_case(mm, oracle, mm.DOUBLE, mm.MULTIPLY, mm.ADD, n, k, m)
    assert oracle.verify(oracle.DOUBLE, c, ref) == -1
    assert max_rel(c, ref) <= TOL["dmma_f64"]


@pytest.mark.parametrize("n,k,m", [(256, 256, 256), (513, 544, 544), (1, 32, 32), (128, 4096, 256), (1024, 1024, 1024)])
def test_half_tensor_path_vs_fp64(mm, oracle, n, k, m):
    """half inputs scaled so that C stays below 65504 (SURVEY.md trap 5); the tensor path keeps
    FP32 accumulators, so it is compared with an FP64 evaluation of the same half inputs."""
    a, b = oracle.fill(oracle.HALF, n, k, m)
    a = (a.astype(np.float32) * np.float32(min(1.0, 500.0 / k))).astype(np.float16)
    c = mm.matrix_multiplication_kernel(a, b, n, k, m, dtype=mm.HALF)
    exact = a.reshape(n, k).astype(np.float64) @ b.reshape(k, m).astype(np.float64)
    assert np.all(np.isfinite(c.astype(np.float32)))
    assert max_rel(c, exact) <= TOL["wgmma_f16"]


def test_half_small_k_against_half_accumulating_oracle(mm, oracle):
    """At K = 32 the oracle's half accumulation is still close: loose agreement with it."""
    a, b, c, ref = run_case(mm, oracle, mm.HALF, mm.MULTIPLY, mm.ADD, 64, 32, 64)
    assert max_rel(c, ref) < 1e-2


@pytest.mark.parametrize("n,k,m,flags", [(512, 1024, 512, 4), (129, 48, 272, 4), (130, 64, 192, 4 | 1)])
def test_float_tf32x3(mm, oracle, n, k, m, flags):
    """MM_FLAG_TF32X3: 3xTF32 split on the tensor cores.  The operand error drops to 2^-22, what
    remains is the tensor core's truncating FP32 accumulation (about K/8 * 3 * 2^-25 relative, biased):
    1.3e-5 observed at K = 1024 against an FP64 evaluation, vs 6e-5 for the single-pass path.
    Tolerance 3e-5."""
    a, b = oracle.fill(oracle.FLOAT, n, k, m)
    c = mm.matrix_multiplication_kernel(a, b, n, k, m, dtype=mm.FLOAT, flags=flags)
    a2 = a.reshape(k, n).T if flags & 1 else a.reshape(n, k)
    exact = a2.astype(np.float64) @ b.reshape(k, m).astype(np.float64)
    assert max_rel(c, exact) <= 3e-5
    ref = oracle.naive(oracle.FLOAT, oracle.MULTIPLY, oracle.ADD, a, b, n, k, m, transposed_a=bool(flags & 1), threads=8)
    assert oracle.verify(oracle.FLOAT, c, ref) == -1


def test_tf32_unbiased(mm, oracle):
    """Round-to-nearest operand preparation keeps the error centred: the MEAN signed relative
    error over C must be far below the 2^-11 a truncating feed would show."""
    a, b, c, ref = run_case(mm, oracle, mm.FLOAT, mm.MULTIPLY, mm.ADD, 512, 1024, 512)
    rel = (c.astype(np.float64) - ref.astype(np.float64)) / ref.astype(np.float64)
    assert abs(float(rel.mean())) < 5e-5


# ---------------------------------------------------------------------------------------------
# 3. CUDA-core semiring path: bit-exact for every type / semiring, ragged shapes included
# ---------------------------------------------------------------------------------------------
def _semiring_cases():
    import gemm_hls_b200 as G
    cases = []
    for dt, w in ((G.FLOAT, 16), (G.DOUBLE, 8), (G.HALF, 32), (G.INT32, 16), (G.UINT32, 16), (G.UINT8, 64)):
        for mp in range(5):
            for rd in range(5):
                cases.append((dt, mp, rd, 65, 2 * w, 3 * w))
    return cases


@pytest.mark.parametrize("dt,mp,rd,n,k,m", _semiring_cases())
def test_semiring_all_combinations_bit_exact(mm, oracle, dt, mp, rd, n, k, m):
    a, b, c, ref = run_case(mm, oracle, dt, mp, rd, n, k, m, flags=mm.FLAG_EXACT, seed=11)
    assert c.tobytes() == ref.tobytes()


SEMIRING_SHAPES = [(256, 256, 256), (513, 528, 528), (1, 64, 64), (127, 64, 192), (300, 1024, 320)]


@pytest.mark.parametrize("n,k,m", SEMIRING_SHAPES)
@pytest.mark.parametrize("dt,mp,rd", [("FLOAT", "ADD", "MIN"), ("FLOAT", "MULTIPLY", "ADD"), ("INT32", "MULTIPLY", "ADD"),
                                      ("DOUBLE", "ADD", "MAX"), ("UINT8", "MULTIPLY", "ADD"), ("HALF", "MULTIPLY", "ADD")])
def test_semiring_shapes_bit_exact(mm, oracle, dt, mp, rd, n, k, m):
    dtype, m_, r_ = getattr(mm, dt), getattr(mm, mp), getattr(mm, rd)
    w = mm.memory_width(dtype)
    k, m = (k + w - 1) // w * w, (m + w - 1) // w * w   # round up to a legal shape for this type
    a, b, c, ref = run_case(mm, oracle, dtype, m_, r_, n, k, m, flags=mm.FLAG_EXACT)
    assert c.tobytes() == ref.tobytes()
    assert oracle.verify(dtype, c, ref) == -1


def test_distance_product_config5_shape_class(mm, oracle):
    """(Add, Min) float — BASELINE config 5's semiring — at 1024^3 against the oracle."""
    a, b, c, ref = run_case(mm, oracle, mm.FLOAT, mm.ADD, mm.MIN, 1024, 1024, 1024)
    assert c.tobytes() == ref.tobytes()


@pytest.mark.parametrize("dt,mp,rd", [("FLOAT", "MULTIPLY", "ADD"), ("DOUBLE", "MULTIPLY", "ADD"), ("HALF", "MULTIPLY", "ADD"),
                                      ("FLOAT", "ADD", "MIN"), ("INT32", "MULTIPLY", "ADD")])
@pytest.mark.parametrize("n,k,m", [(256, 256, 256), (129, 144, 160), (130, 64, 192)])
def test_transposed_a(mm, oracle, dt, mp, rd, n, k, m):
    """MM_TRANSPOSED_A: A stored K x N (include/Utility.h:31-35)."""
    dtype, m_, r_ = getattr(mm, dt), getattr(mm, mp), getattr(mm, rd)
    if k % mm.memory_width(dtype) or m % mm.memory_width(dtype):
        pytest.skip("shape not legal for this data type")
    a, b = oracle.fill(dtype, n, k, m, 9)
    if dtype == mm.HALF:
        a = (a.astype(np.float32) * np.float32(0.25)).astype(np.float16)
    exact = mm.matrix_multiplication_kernel(a, b, n, k, m, dtype=dtype, map_op=m_, reduce_op=r_,
                                            flags=mm.FLAG_TRANSPOSED_A | mm.FLAG_EXACT)
    ref = oracle.naive(dtype, m_, r_, a, b, n, k, m, transposed_a=True, threads=8)
    assert exact.tobytes() == ref.tobytes()
    fast = mm.matrix_multiplication_kernel(a, b, n, k, m, dtype=dtype, map_op=m_, reduce_op=r_,
                                           flags=mm.FLAG_TRANSPOSED_A)
    path = mm.kernel_path(dtype, m_, r_, mm.FLAG_TRANSPOSED_A)
    if path == "semiring_simt":
        assert fast.tobytes() == ref.tobytes()
    elif dtype == mm.HALF:
        e64 = a.reshape(k, n).astype(np.float64).T @ b.reshape(k, m).astype(np.float64)
        assert max_rel(fast, e64) <= TOL[path]
    else:
        assert max_rel(fast, ref) <= TOL[path]


# ---------------------------------------------------------------------------------------------
# 4. the device-resident lifecycle (RunHardware's call sequence) and error behaviour
# ---------------------------------------------------------------------------------------------
def test_context_lifecycle_matches_runhardware_sequence(mm, oracle):
    """MakeBuffer x3, CopyFromHost x3, MakeKernel+ExecuteTask, CopyToHost (host/RunHardware.cpp:116-190)."""
    n, k, m = 384, 256, 512
    a, b = oracle.fill(oracle.FLOAT, n, k, m)
    ref = oracle.naive(oracle.FLOAT, oracle.MULTIPLY, oracle.ADD, a, b, n, k, m, threads=8)
    with mm.Context(0) as ctx:
        da, db, dc = ctx.alloc(a.nbytes), ctx.alloc(b.nbytes), ctx.alloc(n * m * 4)
        ctx.copy_to_device(da, a)
        ctx.copy_to_device(db, b)
        ctx.copy_to_device(dc, np.zeros(n * m, np.float32))
        sec_dev, sec_wall = ctx.execute(mm.FLOAT, mm.MULTIPLY, mm.ADD, da, db, dc, n, k, m)
        assert 0 < sec_dev <= sec_wall
        c = np.empty((n, m), np.float32)
        ctx.copy_to_host(c, dc)
        # executing twice gives the same bits (C is output-only, fully overwritten)
        ctx.execute(mm.FLOAT, mm.MULTIPLY, mm.ADD, da, db, dc, n, k, m)
        c2 = np.empty((n, m), np.float32)
        ctx.copy_to_host(c2, dc)
        for p in (da, db, dc):
            ctx.free(p)
    assert oracle.verify(oracle.FLOAT, c, ref) == -1
    assert c.tobytes() == c2.tobytes()


def test_shape_errors_match_reference_wording(mm):
    with pytest.raises(mm.MMError) as e:
        mm.matrix_multiplication_kernel(np.ones(32 * 40, np.float32), np.ones(40 * 32, np.float32), 32, 40, 32)
    assert "K (40) must be divisable by the memory width in K (16)." in str(e.value)


def test_row_block_split_equals_single_launch(mm, oracle):
    """Row-blocks of C are independent (SURVEY.md section 8e): computing two row-blocks separately
    and concatenating must equal the single launch bit for bit — the multi-GPU partition invariant."""
    n, k, m = 512, 512, 512
    a, b = oracle.fill(oracle.FLOAT, n, k, m)
    whole = mm.matrix_multiplication_kernel(a, b, n, k, m)
    a2 = a.reshape(n, k)
    top = mm.matrix_multiplication_kernel(a2[:256], b, 256, k, m)
    bot = mm.matrix_multiplication_kernel(a2[256:], b, 256, k, m)
    assert np.concatenate([top, bot]).tobytes() == whole.tobytes()


# ---------------------------------------------------------------------------------------------
# 5. streams and graphs: the asynchronous entry on a caller-owned stream, CUDA-graph capture
# ---------------------------------------------------------------------------------------------
def test_enqueue_on_caller_stream_and_graph_replay(mm, oracle):
    """mm_kernel_enqueue on a caller-owned stream is capturable into a CUDA graph once the context's
    scratch exists (first call outside capture); replaying the graph recomputes C from new A."""
    torch = pytest.importorskip("torch")
    n, k, m = 384, 512, 640
    a, b = oracle.fill(oracle.FLOAT, n, k, m)
    ref = oracle.naive(oracle.FLOAT, oracle.MULTIPLY, oracle.ADD, a, b, n, k, m, threads=8)
    dev = torch.device("cuda", 0)
    ta = torch.from_numpy(a.reshape(n, k)).to(dev)
    tb = torch.from_numpy(b.reshape(k, m)).to(dev)
    tc = torch.zeros((n, m), device=dev, dtype=torch.float32)
    with mm.Context(0) as ctx:
        s = torch.cuda.Stream(device=dev)
        with torch.cuda.stream(s):
            ctx.enqueue(mm.FLOAT, mm.MULTIPLY, mm.ADD, ta.data_ptr(), tb.data_ptr(), tc.data_ptr(), n, k, m,
                        stream=s.cuda_stream)          # warm-up: allocates the scratch, loads the kernels
        s.synchronize()
        assert oracle.verify(oracle.FLOAT, tc.cpu().numpy(), ref) == -1
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            ctx.enqueue(mm.FLOAT, mm.MULTIPLY, mm.ADD, ta.data_ptr(), tb.data_ptr(), tc.data_ptr(), n, k, m,
                        stream=torch.cuda.current_stream().cuda_stream)
        ta.mul_(2.0)                                    # new input, same buffers
        tc.zero_()
        g.replay()
        torch.cuda.synchronize()
        got = tc.cpu().numpy()
    assert oracle.verify(oracle.FLOAT, got, (2.0 * ref).astype(np.float32)) == -1


def test_two_contexts_on_two_streams_do_not_interfere(mm, oracle):
    """Contexts own their scratch: two contexts running different problems back to back on their
    own streams give the same bits as running alone."""
    shapes = [(256, 512, 384, mm.FLOAT, mm.MULTIPLY, mm.ADD), (200, 256, 512, mm.FLOAT, mm.ADD, mm.MIN)]
    alone, data = [], []
    for n, k, m, dt, mp, rd in shapes:
        a, b = oracle.fill(dt, n, k, m, 21)
        data.append((a, b))
        alone.append(mm.matrix_multiplication_kernel(a, b, n, k, m, dtype=dt, map_op=mp, reduce_op=rd))
    ctxs = [mm.Context(0), mm.Context(0)]
    try:
        outs = []
        for rep in range(3):
            outs = [ctxs[i].gemm_host(dt, mp, rd, data[i][0], data[i][1], n, k, m)[0]
                    for i, (n, k, m, dt, mp, rd) in enumerate(shapes)]
        for o, ref in zip(outs, alone):
            assert o.tobytes() == ref.tobytes()
    finally:
        for c in ctxs:
            c.close()
