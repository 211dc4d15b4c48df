"""gemm_hls_b200 — H100-native (sm_90a) MatrixMultiplication hot path of spcl/gemm_hls.

Thin ctypes binding over the C-ABI library ``libmm_b200.so`` (include/mm_b200.h).  The product is
the CUDA library; this module only loads it and passes pointers.  There is no CPU fallback: if the
library is missing or no H100 is present the calls raise.

Reference surface mirrored here (file:line under the reference checkout):
  * ``MatrixMultiplicationKernel(a, b, c, n, k, m)``  include/MatrixMultiplication.h:155-171
      -> :func:`matrix_multiplication_kernel` (host arrays in, host array out)
  * ``hlslib::ocl::Context`` / ``MakeBuffer`` / ``CopyFromHost`` / ``MakeKernel`` / ``ExecuteTask``
      host/RunHardware.cpp:116-190  -> :class:`Context`
"""
import ctypes
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
# MM_B200_LIB: A/B experiments load a variant build of the library; the product is the in-tree library
LIB_PATH = os.environ.get("MM_B200_LIB") or os.path.join(HERE, "libmm_b200.so")

# MM_DATA_TYPE codes (BFLOAT16 is a library-level extension: the reference has no such type)
HALF, FLOAT, DOUBLE, INT32, UINT32, UINT8, BFLOAT16 = range(7)
# MM_MAP_OP / MM_REDUCE_OP codes (hlslib::op functors)
MULTIPLY, ADD, MIN, MAX, AND = range(5)
# flags
FLAG_NONE, FLAG_TRANSPOSED_A, FLAG_EXACT, FLAG_TF32X3 = 0, 1, 2, 4
FLAG_BATCH_SHARED_A, FLAG_BATCH_SHARED_B = 8, 16   # batched calls: every problem reads the same A / B
WITNESS_NONE = 0xFFFFFFFF   # MM_WITNESS_NONE: the reduction never selected a term (Context.enqueue_witness)

# numpy has no bfloat16: BFLOAT16 host arrays are its bit patterns (np.uint16, or ml_dtypes.bfloat16), taken by view
NP_DTYPE = {HALF: np.float16, FLOAT: np.float32, DOUBLE: np.float64,
            INT32: np.int32, UINT32: np.uint32, UINT8: np.uint8, BFLOAT16: np.uint16}
DTYPE_FROM_NAME = {"half": HALF, "float": FLOAT, "double": DOUBLE, "int": INT32,
                   "unsigned": UINT32, "unsigned int": UINT32, "uint8_t": UINT8, "bfloat16": BFLOAT16}
OP_FROM_NAME = {"Multiply": MULTIPLY, "Product": MULTIPLY, "Add": ADD, "Sum": ADD,
                "Min": MIN, "Max": MAX, "And": AND}

# MM_TUNE_* knobs (include/mm_b200.h)
(TUNE_CTA_GROUP, TUNE_BLOCK_N, TUNE_STAGES, TUNE_RASTER_ROWS, TUNE_TILE_SYNC, TUNE_B_MN, TUNE_L2_POLICY,
 TUNE_B_OVERLAP, TUNE_TMA_STORE, TUNE_DMMA_TILE_ROWS, TUNE_EXPERIMENT_TF32_NO_ROUND, TUNE_SEMIRING_RING) = range(12)
TUNE_NAMES = {"cta_group": TUNE_CTA_GROUP, "block_n": TUNE_BLOCK_N, "stages": TUNE_STAGES,
              "raster_rows": TUNE_RASTER_ROWS, "tile_sync": TUNE_TILE_SYNC, "b_mn": TUNE_B_MN,
              "l2_policy": TUNE_L2_POLICY, "b_overlap": TUNE_B_OVERLAP, "tma_store": TUNE_TMA_STORE,
              "dmma_tile_rows": TUNE_DMMA_TILE_ROWS, "tf32_no_round": TUNE_EXPERIMENT_TF32_NO_ROUND,
              "semiring_ring": TUNE_SEMIRING_RING}

EXPORTS = ["mm_last_error", "mm_version", "mm_dtype_size", "mm_memory_width", "mm_context_create",
           "mm_context_destroy", "mm_buffer_alloc", "mm_buffer_free", "mm_copy_to_device",
           "mm_copy_to_host", "mm_kernel_execute", "mm_kernel_enqueue", "mm_kernel_launch_count",
           "mm_kernel_path", "mm_gemm_host", "mm_context_set_profiling", "mm_context_profile_read",
           "mm_context_set_tuning", "mm_context_get_tuning", "mm_context_reserve",
           "mm_kernel_enqueue_batched", "mm_context_reserve_batched", "mm_kernel_enqueue_witness",
           "mm_kernel_enqueue_accumulate", "mm_multi_create", "mm_multi_destroy", "mm_multi_device_count",
           "mm_multi_context", "mm_multi_peer_access", "mm_multi_partition", "mm_multi_gemm_host", "mm_multi_upload",
           "mm_multi_execute", "mm_multi_download", "mm_kernel_enqueue_closure", "mm_closure_block",
           "mm_kernel_enqueue_bool", "mm_kernel_enqueue_bool_closure"]


class MMError(RuntimeError):
    """Counterpart of hlslib::ocl::RuntimeError / ConfigurationError (common/OpenCL.h:99-157)."""

    def __init__(self, code, message):
        super().__init__("mm_b200 error %d: %s" % (code, message))
        self.code = code


_lib = None


def lib():
    """Load libmm_b200.so; raises if it has not been built (python gemm_hls_b200/build.py)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise MMError(-1, "%s not found — build it with `python gemm_hls_b200/build.py` "
                              "(there is no CPU fallback)" % LIB_PATH)
        L = ctypes.CDLL(LIB_PATH)
        vp, i, u, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint, ctypes.c_size_t
        dp = ctypes.POINTER(ctypes.c_double)
        L.mm_last_error.restype = ctypes.c_char_p
        L.mm_dtype_size.argtypes, L.mm_dtype_size.restype = [i], sz
        L.mm_memory_width.argtypes, L.mm_memory_width.restype = [i], u
        L.mm_context_create.argtypes = [i, ctypes.POINTER(vp)]
        L.mm_context_destroy.argtypes = [vp]
        L.mm_buffer_alloc.argtypes = [vp, sz, ctypes.POINTER(vp)]
        L.mm_buffer_free.argtypes = [vp, vp]
        L.mm_copy_to_device.argtypes = [vp, vp, vp, sz]
        L.mm_copy_to_host.argtypes = [vp, vp, vp, sz]
        L.mm_kernel_execute.argtypes = [vp, i, i, i, i, vp, vp, vp, u, u, u, dp, dp]
        L.mm_kernel_enqueue.argtypes = [vp, i, i, i, i, vp, vp, vp, u, u, u, vp]
        L.mm_kernel_launch_count.argtypes = [i, i, i, i]
        L.mm_kernel_path.argtypes, L.mm_kernel_path.restype = [i, i, i, i], ctypes.c_char_p
        L.mm_gemm_host.argtypes = [vp, i, i, i, i, vp, vp, vp, u, u, u, dp, dp]
        L.mm_context_set_profiling.argtypes = [vp, i]
        L.mm_context_profile_read.argtypes = [vp, dp, dp, ctypes.POINTER(i)]
        L.mm_context_set_tuning.argtypes = [vp, i, i]
        L.mm_context_get_tuning.argtypes = [vp, i, ctypes.POINTER(i)]
        L.mm_context_reserve.argtypes = [vp, i, i, u, u, u]
        L.mm_kernel_enqueue_batched.argtypes = [vp, i, i, i, i, vp, vp, vp, u, u, u, u, vp]
        L.mm_context_reserve_batched.argtypes = [vp, i, i, u, u, u, u]
        L.mm_kernel_enqueue_witness.argtypes = [vp, i, i, i, i, vp, vp, vp, vp, u, u, u, u, vp]
        L.mm_kernel_enqueue_accumulate.argtypes = [vp, i, i, i, i, vp, vp, vp, u, u, u, u, vp]
        L.mm_kernel_enqueue_closure.argtypes = [vp, i, i, i, i, vp, u, u, vp]
        L.mm_closure_block.argtypes, L.mm_closure_block.restype = [i], u
        L.mm_kernel_enqueue_bool.argtypes = [vp, i, vp, vp, vp, u, u, u, u, vp]
        L.mm_kernel_enqueue_bool_closure.argtypes = [vp, i, vp, u, u, vp]
        L.mm_multi_create.argtypes = [i, ctypes.POINTER(i), ctypes.POINTER(vp)]
        L.mm_multi_destroy.argtypes = [vp]
        L.mm_multi_device_count.argtypes = [vp]
        L.mm_multi_context.argtypes, L.mm_multi_context.restype = [vp, i], vp
        L.mm_multi_peer_access.argtypes = [vp]
        up = ctypes.POINTER(u)
        L.mm_multi_partition.argtypes = [i, i, u, u, up, up, up, up]
        L.mm_multi_gemm_host.argtypes = [vp, i, i, i, i, vp, vp, vp, u, u, u, dp, dp]
        L.mm_multi_upload.argtypes = [vp, i, i, vp, vp, u, u, u]
        L.mm_multi_execute.argtypes = [vp, i, i, i, i, u, u, u, dp, dp]
        L.mm_multi_download.argtypes = [vp, i, vp, u, u]
        _lib = L
    return _lib


def _check(rc):
    if rc != 0:
        raise MMError(rc, lib().mm_last_error().decode())


def memory_width(dtype):
    return int(lib().mm_memory_width(dtype))


def closure_block(dtype):
    """b of Context.enqueue_closure: the width of its blocks of indices (0 for an unknown dtype)."""
    return int(lib().mm_closure_block(dtype))


def kernel_path(dtype, map_op=MULTIPLY, reduce_op=ADD, flags=0):
    return lib().mm_kernel_path(dtype, map_op, reduce_op, flags).decode()


def launch_count(dtype, map_op=MULTIPLY, reduce_op=ADD, flags=0):
    return int(lib().mm_kernel_launch_count(dtype, map_op, reduce_op, flags))


class Context:
    """Device context: the hlslib::ocl::Context + Program + Kernel of host/RunHardware.cpp:116-162."""

    def __init__(self, device=0):
        self._h = ctypes.c_void_p()
        _check(lib().mm_context_create(device, ctypes.byref(self._h)))
        self.device = device

    def close(self):
        if self._h:
            lib().mm_context_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # Context::MakeBuffer
    def alloc(self, nbytes):
        p = ctypes.c_void_p()
        _check(lib().mm_buffer_alloc(self._h, nbytes, ctypes.byref(p)))
        return p.value

    def free(self, dptr):
        _check(lib().mm_buffer_free(self._h, dptr))

    # Buffer::CopyFromHost / CopyToHost
    def copy_to_device(self, dptr, host_array):
        host_array = np.ascontiguousarray(host_array)
        _check(lib().mm_copy_to_device(self._h, dptr, host_array.ctypes.data, host_array.nbytes))

    def copy_to_host(self, host_array, dptr):
        assert host_array.flags["C_CONTIGUOUS"]
        _check(lib().mm_copy_to_host(self._h, host_array.ctypes.data, dptr, host_array.nbytes))

    # Kernel::ExecuteTask -> (seconds_device, seconds_wall)
    def execute(self, dtype, map_op, reduce_op, a_dev, b_dev, c_dev, n, k, m, flags=0):
        sd, sw = ctypes.c_double(), ctypes.c_double()
        _check(lib().mm_kernel_execute(self._h, dtype, map_op, reduce_op, flags, a_dev, b_dev, c_dev,
                                       n, k, m, ctypes.byref(sd), ctypes.byref(sw)))
        return sd.value, sw.value

    def enqueue(self, dtype, map_op, reduce_op, a_dev, b_dev, c_dev, n, k, m, flags=0, stream=None):
        """Asynchronous launch on a CUDA stream handle (int, e.g. torch's stream.cuda_stream)."""
        _check(lib().mm_kernel_enqueue(self._h, dtype, map_op, reduce_op, flags, a_dev, b_dev, c_dev,
                                       n, k, m, ctypes.c_void_p(stream) if stream else None))

    def enqueue_batched(self, dtype, map_op, reduce_op, a_dev, b_dev, c_dev, n, k, m, batch, flags=0, stream=None):
        """`batch` packed problems (A at a + i*n*k, B at b + i*k*m unless FLAG_BATCH_SHARED_A / _B, C at
        c + i*n*m elements) in one asynchronous launch sequence; each C equals its single enqueue bit for bit."""
        _check(lib().mm_kernel_enqueue_batched(self._h, dtype, map_op, reduce_op, flags, a_dev, b_dev, c_dev,
                                               n, k, m, batch, ctypes.c_void_p(stream) if stream else None))

    def enqueue_witness(self, dtype, map_op, reduce_op, a_dev, b_dev, c_dev, w_dev, n, k, m, batch=1, flags=0,
                        stream=None):
        """C exactly as enqueue_batched computes it, plus W (n*m uint32 per problem, packed like C): for a Min or
        Max reduce, the k whose term each element of C was selected from last, or WITNESS_NONE (include/mm_b200.h)."""
        _check(lib().mm_kernel_enqueue_witness(self._h, dtype, map_op, reduce_op, flags, a_dev, b_dev, c_dev, w_dev,
                                               n, k, m, batch, ctypes.c_void_p(stream) if stream else None))

    def enqueue_accumulate(self, dtype, map_op, reduce_op, a_dev, b_dev, c_dev, n, k, m, batch=1, flags=0,
                           stream=None):
        """C <- R(C, P) in place: P is what enqueue_batched would write with the same arguments, R one application of
        the call's reduce with the old C first (include/mm_b200.h).  C must not overlap A or B."""
        _check(lib().mm_kernel_enqueue_accumulate(self._h, dtype, map_op, reduce_op, flags, a_dev, b_dev, c_dev,
                                                  n, k, m, batch, ctypes.c_void_p(stream) if stream else None))

    def enqueue_closure(self, dtype, map_op, reduce_op, d_dev, n, batch=1, flags=0, stream=None):
        """D <- its closure over (map_op, reduce_op) in place, for `batch` packed n x n problems (reduce Min or Max):
        blocked Floyd-Warshall with blocks of closure_block(dtype) indices, in the order include/mm_b200.h states.
        The diagonal is not initialised."""
        _check(lib().mm_kernel_enqueue_closure(self._h, dtype, map_op, reduce_op, flags, d_dev, n, batch,
                                               ctypes.c_void_p(stream) if stream else None))

    def enqueue_bool(self, a_dev, b_dev, c_dev, n, k, m, batch=1, flags=0, stream=None):
        """Bit-packed Boolean product C = A . B (C[i][j] = OR_k A[i][k] AND B[k][j]) for `batch` packed problems, on the
        b1 tensor cores.  Each matrix is row-major with bit j % 8 of byte j / 8 for column j (numpy.packbits(...,
        bitorder='little')); k and m must be multiples of 128."""
        _check(lib().mm_kernel_enqueue_bool(self._h, flags, a_dev, b_dev, c_dev, n, k, m, batch,
                                            ctypes.c_void_p(stream) if stream else None))

    def enqueue_bool_closure(self, d_dev, n, batch=1, flags=0, stream=None):
        """D <- its transitive closure (paths of one or more edges) in place, for `batch` packed bit-packed n x n
        matrices (layout as enqueue_bool; n a multiple of 128).  The diagonal is not set reflexively."""
        _check(lib().mm_kernel_enqueue_bool_closure(self._h, flags, d_dev, n, batch,
                                                    ctypes.c_void_p(stream) if stream else None))

    def set_tuning(self, **knobs):
        """mm_context_set_tuning by name, e.g. ctx.set_tuning(cta_group=1, stages=4)."""
        for name, value in knobs.items():
            _check(lib().mm_context_set_tuning(self._h, TUNE_NAMES[name], int(value)))

    def get_tuning(self, name):
        v = ctypes.c_int()
        _check(lib().mm_context_get_tuning(self._h, TUNE_NAMES[name], ctypes.byref(v)))
        return v.value

    def reserve(self, dtype, n, k, m, flags=0):
        _check(lib().mm_context_reserve(self._h, dtype, flags, n, k, m))

    def reserve_batched(self, dtype, n, k, m, batch, flags=0):
        _check(lib().mm_context_reserve_batched(self._h, dtype, flags, n, k, m, batch))

    def set_profiling(self, enable=True):
        _check(lib().mm_context_set_profiling(self._h, int(enable)))

    def profile_read(self):
        """(prep_seconds_sum, main_kernel_seconds_sum, calls) since the last read."""
        p, mn, c = ctypes.c_double(), ctypes.c_double(), ctypes.c_int()
        _check(lib().mm_context_profile_read(self._h, ctypes.byref(p), ctypes.byref(mn), ctypes.byref(c)))
        return p.value, mn.value, c.value

    def gemm_host(self, dtype, map_op, reduce_op, a, b, n, k, m, flags=0, out=None):
        """Host arrays in, host array out (H2D, kernel, D2H); returns (C, seconds_device, seconds_wall)."""
        return _gemm_host(self._h, dtype, map_op, reduce_op, a, b, n, k, m, flags, out)


def multi_partition(n_gpus, index, n, k):
    """(row_begin, row_end, b_row_begin, b_row_end) of GPU `index` in an n_gpus split (mm_multi_partition; no device needed)."""
    out = [ctypes.c_uint() for _ in range(4)]
    _check(lib().mm_multi_partition(n_gpus, index, n, k, *[ctypes.byref(o) for o in out]))
    return tuple(o.value for o in out)


class _BorrowedContext(Context):
    """A per-device context owned by a Multi (never destroyed from Python)."""

    def __init__(self, handle, device):
        self._h = ctypes.c_void_p(handle)
        self.device = device

    def close(self):
        self._h = ctypes.c_void_p()


class Multi:
    """C row-blocks over G GPUs of this process (mm_multi_*, SURVEY.md section 8e): one blocking call on
    host arrays, or the device-resident upload / execute / download lifecycle of RunHardware."""

    def __init__(self, n_gpus, devices=None):
        self._h = ctypes.c_void_p()
        dev = (ctypes.c_int * n_gpus)(*devices) if devices is not None else None
        _check(lib().mm_multi_create(n_gpus, dev, ctypes.byref(self._h)))
        self.n_gpus = n_gpus

    def close(self):
        if self._h:
            lib().mm_multi_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def peer_access(self):
        return bool(lib().mm_multi_peer_access(self._h))

    def context(self, index):
        return _BorrowedContext(lib().mm_multi_context(self._h, index), index)

    def set_tuning(self, **knobs):
        for g in range(self.n_gpus):
            self.context(g).set_tuning(**knobs)

    def gemm_host(self, dtype, map_op, reduce_op, a, b, n, k, m, flags=0, out=None):
        return _gemm_host(self._h, dtype, map_op, reduce_op, a, b, n, k, m, flags, out, fn=lib().mm_multi_gemm_host)

    def upload(self, dtype, a, b, n, k, m, flags=0):
        a = _host_operand(dtype, a)
        b = _host_operand(dtype, b)
        _check(lib().mm_multi_upload(self._h, dtype, flags, a.ctypes.data, b.ctypes.data, n, k, m))

    def execute(self, dtype, map_op, reduce_op, n, k, m, flags=0):
        sd, sw = ctypes.c_double(), ctypes.c_double()
        _check(lib().mm_multi_execute(self._h, dtype, map_op, reduce_op, flags, n, k, m, ctypes.byref(sd), ctypes.byref(sw)))
        return sd.value, sw.value

    def download(self, dtype, n, m, out=None):
        """C of the last execute into `out` (a C-contiguous array of n*m elements of the type), or a new array."""
        if out is None:
            out = np.empty((n, m), dtype=NP_DTYPE[dtype])
        elif not out.flags["C_CONTIGUOUS"] or out.nbytes != n * m * int(lib().mm_dtype_size(dtype)):
            raise MMError(1, "out must be a C-contiguous array of n*m elements of the type")
        _check(lib().mm_multi_download(self._h, dtype, out.ctypes.data, n, m))
        return out


def _host_operand(dtype, x):
    """x as the flat contiguous host array the library reads.  BFLOAT16 takes any 2-byte array that is not a
    floating-point numpy type (np.uint16 bit patterns, ml_dtypes.bfloat16) as it is: its bytes are the
    bfloat16 values.  A float array would need a rounding the caller did not ask for, so it is refused."""
    if dtype == BFLOAT16:
        x = np.asarray(x)
        if x.dtype.itemsize != 2 or x.dtype.kind == "f":
            raise MMError(1, "BFLOAT16 takes bfloat16 bit patterns (np.uint16 or ml_dtypes.bfloat16 arrays), "
                             "not %s: convert explicitly" % x.dtype)
        return np.ascontiguousarray(x).reshape(-1)
    return np.ascontiguousarray(x, dtype=NP_DTYPE.get(dtype)).reshape(-1)


def _gemm_host(handle, dtype, map_op, reduce_op, a, b, n, k, m, flags, out, fn=None):
    npdt = NP_DTYPE.get(dtype)  # unknown codes are rejected by the library itself (MM_ERR_INVALID)
    a = _host_operand(dtype, a)
    b = _host_operand(dtype, b)
    if dtype == BFLOAT16:
        npdt = a.dtype  # C comes back with A's dtype
    if npdt is not None and (a.size != n * k or b.size != k * m):
        raise MMError(1, "A must hold n*k and B k*m elements")
    c = out if out is not None else np.empty((n, m), dtype=npdt if npdt is not None else a.dtype)
    sd, sw = ctypes.c_double(), ctypes.c_double()
    _check((fn or lib().mm_gemm_host)(handle, dtype, map_op, reduce_op, flags, a.ctypes.data, b.ctypes.data,
                                      c.ctypes.data, n, k, m, ctypes.byref(sd), ctypes.byref(sw)))
    return c, sd.value, sw.value


def matrix_multiplication_kernel(a, b, n, k, m, dtype=FLOAT, map_op=MULTIPLY, reduce_op=ADD, flags=0, out=None):
    """The reference's ``MatrixMultiplicationKernel(a, b, c, n, k, m)`` called with host pointers
    (test/TestSimulation.cpp:66), for a run-time chosen (MM_DATA_TYPE, MM_MAP_OP, MM_REDUCE_OP).
    Returns C as an (n, m) numpy array (`out`, the reference's c, when given).  Uses the library's
    default context on device 0."""
    c, _, _ = _gemm_host(None, dtype, map_op, reduce_op, a, b, n, k, m, flags, out)
    return c
