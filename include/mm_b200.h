/* mm_b200.h — C-ABI of libmm_b200.so: the H100-native (sm_90a) MatrixMultiplication hot path.
 *
 * This is the drop-in boundary for ONE path of spcl/gemm_hls: the tiled matrix-multiplication
 * kernel  C[N x M] = A[N x K] (x) B[K x M]  over an (OperatorMap, OperatorReduce) semiring
 * (reference: kernel/Top.cpp:9-117 -> kernel/Memory.cpp streamers -> kernel/Compute.cpp PE chain).
 * Every entry point below names the reference interface it replaces (file:line under the
 * reference checkout).  Plain pointers and sizes only; no C++/torch types cross this line.
 *
 * Layouts (identical to the reference, include/Utility.h:27-39): A row-major N x K (K x N when
 * MM_FLAG_TRANSPOSED_A), B row-major K x M, C row-major N x M, dense, no leading dimensions.
 * The reference's MemoryPack*_t arrays are bit-identical to flat Data_t arrays
 * (include/Utility.h:44-63), so flat pointers are passed here.
 *
 * Error handling: every function returns MM_OK (0) or an MM_ERR_* code; mm_last_error() gives the
 * message for the calling thread.  The library never exits the process and never falls back to a
 * CPU implementation: without a usable CUDA device every compute entry point fails with
 * MM_ERR_CUDA.
 */
#ifndef MM_B200_H_
#define MM_B200_H_

#include <stddef.h>

#if defined(__GNUC__)
#define MM_API __attribute__((visibility("default")))
#else
#define MM_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

/* MM_DATA_TYPE (reference CMakeLists.txt:16, include/Config.h.in:15). */
enum {
  MM_DTYPE_HALF = 0,   /* "half"      IEEE binary16 */
  MM_DTYPE_FLOAT = 1,  /* "float"  */
  MM_DTYPE_DOUBLE = 2, /* "double" */
  MM_DTYPE_INT32 = 3,  /* "int"    */
  MM_DTYPE_UINT32 = 4, /* "unsigned" */
  MM_DTYPE_UINT8 = 5,  /* "uint8_t" (reference CMakeLists.txt:43-46) */
  MM_DTYPE_BFLOAT16 = 6, /* bfloat16 (8-bit exponent, 8-bit significand): a library-level extension; the
                          * reference has no such type.  Size 2, memory width 32, as half. */
  MM_DTYPE_COUNT = 7
};

/* MM_MAP_OP / MM_REDUCE_OP = hlslib::op functors (hlslib/include/hlslib/xilinx/Operators.h:20-100).
 * identity(): Add 0, Multiply 1, And true, Min numeric_limits<T>::max(),
 * Max numeric_limits<T>::min() (the smallest POSITIVE value for floating point — reproduced). */
enum {
  MM_OP_MULTIPLY = 0, /* hlslib::op::Multiply == Product */
  MM_OP_ADD = 1,      /* hlslib::op::Add == Sum */
  MM_OP_MIN = 2,
  MM_OP_MAX = 3,
  MM_OP_AND = 4,
  MM_OP_COUNT = 5
};

/* Flags for the execute calls. */
enum {
  MM_FLAG_NONE = 0,
  /* A is stored K x N (reference MM_TRANSPOSED_A, CMakeLists.txt:30, include/Utility.h:31-35). */
  MM_FLAG_TRANSPOSED_A = 1,
  /* Force the CUDA-core semiring kernel also for (Multiply, Add), and the literal C++ Min / Max for
   * float.  That kernel accumulates each C element sequentially over k in Data_t with one rounding
   * per Map and per Reduce (no FMA contraction), i.e. it is BIT-IDENTICAL to the reference's Naive<>
   * / FPGA datapath for every data type and every input, including NaN and signed zeros.
   * Without the flag:
   *   - float  (Multiply, Add): tf32 wgmma, operands rounded to nearest TF32 (10-bit
   *     mantissa), FP32 accumulation.  Meets the reference's 1e-3 relative criterion for SAME-SIGN
   *     data such as its own U[1,10] inputs (measured <= 2.1e-4); for mixed-sign data the error is
   *     bounded relative to sum|a*b|, not to |sum a*b| — use MM_FLAG_TF32X3 or MM_FLAG_EXACT there.
   *   - double (Multiply, Add): DMMA, FP64 throughout; differs from Naive<> only by summation order
   *     (measured <= 1e-14 relative).
   *   - half   (Multiply, Add): f16 wgmma with FP32 accumulation and ONE rounding to half at
   *     the end.  The reference (Naive<half>, and its FPGA datapath) accumulates IN HALF, so this
   *     path is closer to the exact product than the reference is and does NOT reproduce the
   *     reference's rounding: against Naive<half> on U[1,10] inputs 15 % of the elements differ by
   *     more than 1e-3 at K = 32 and 63 % at K = 544.  The reference's TestSimulation compares half
   *     EXACTLY (test/TestSimulation.cpp:79-85), so the host executables of this project build half
   *     with MM_FLAG_EXACT unless configured with -DMM_HALF_TENSOR=ON (INTEGRATION.md section 3).
   *   - bfloat16 (Multiply, Add): bf16 wgmma with FP32 accumulation and ONE rounding to bfloat16 at the
   *     end (round to nearest even).  Unlike a Naive<bfloat16>, it does not accumulate in bfloat16.  Under
   *     MM_FLAG_EXACT, and for every other semiring, bfloat16 is BIT-IDENTICAL to a Naive<> that rounds to
   *     bfloat16 after every Map and every Reduce.  Min / Max are the literal `(a < b) ? a : b`, as for half.
   *     MM_FLAG_TF32X3 and the tf32_no_round knob do not apply.
   *   - uint8_t (Multiply, Add): u8 wgmma, exact 32-bit integer accumulation, low byte stored — BIT-IDENTICAL
   *     to the reference's modulo-256 arithmetic.  Used for K <= 33024 (255^2 * K < 2^31); the CUDA-core kernel beyond.
   *   - float Min / Max (as Map or Reduce): the hardware FMNMX.  Identical to the reference's
   *     `(a < b) ? a : b` for all finite inputs except that a tie between -0 and +0 yields -0 for Min
   *     (+0 for Max) where the reference returns the second operand, and NaN operands are dropped
   *     where the reference's comparison lets a NaN in the SECOND operand through.  Inputs without
   *     NaN and without negative zeros (or products / sums that produce them) are bit-identical. */
  MM_FLAG_EXACT = 2,
  /* float (Multiply, Add) on the tensor cores with the 3xTF32 split (hi*hi + hi*lo + lo*hi, each
   * operand split into two TF32 values): ~FP32 accuracy (about 1e-6 relative) at 1/3 of the TF32
   * rate.  Ignored for every other configuration.  Per element, |C - A'B'| <= half an ulp of C +
   * 0.25 * 3K * 2^-23 * sum|a'*b'| over the split operands; on an H100 the worst case seen needed 0.042
   * in place of 0.25 (same-sign data, K up to 16384).
   *
   * Every tensor-core path (TF32, 3xTF32, half, bfloat16, DMMA) propagates +-inf and NaN as IEEE arithmetic
   * on the prepared operands does: inf * x = +-inf, inf - inf and inf * 0 = NaN.  Operand preparation
   * never overflows: a finite float that rounds past the largest TF32 value saturates to +-0x7F7FE000
   * (|x| >= 3.40199e38), so C stays finite where the exact product is.  Subnormal operands are kept, not
   * flushed, by the tf32, f16 and bf16 tensor cores (measured on an H100). */
  MM_FLAG_TF32X3 = 4,
  /* Two flags, meaningful only in batched calls (mm_kernel_enqueue_batched).  The single-problem
   * entries ignore them: a single call is a batch of one, so the statement holds trivially. */
  MM_FLAG_BATCH_SHARED_A = 8,  /* every problem of the batch reads the same A */
  MM_FLAG_BATCH_SHARED_B = 16  /* every problem of the batch reads the same B */
};

enum {
  MM_OK = 0,
  MM_ERR_INVALID = 1, /* bad argument (null pointer, unknown dtype/op, zero size) */
  MM_ERR_SHAPE = 2,   /* K or M not divisible by the memory width (host/RunHardware.cpp:50-61) */
  MM_ERR_CUDA = 3,    /* CUDA runtime / driver failure, or no device */
  MM_ERR_NOMEM = 4,   /* device allocation failed */
  MM_ERR_UNSUPPORTED = 5
};

/* Opaque device context.  Replaces hlslib::ocl::Context + Program + Kernel
 * (hlslib/include/hlslib/common/OpenCL.h:366-500, host/RunHardware.cpp:116-154): owns the CUDA
 * device binding, one stream, timing events and the scratch the tensor-core path needs. */
typedef struct mm_context mm_context;

/* Message for the last failing call on this thread (never NULL).  Replaces the what() of
 * hlslib::ocl::{ConfigurationError,RuntimeError} (common/OpenCL.h:99-157). */
MM_API const char *mm_last_error(void);

/* Size in bytes of one element of `dtype` (0 if unknown).  Reference: sizeof(Data_t). */
MM_API size_t mm_dtype_size(int dtype);

/* Elements per 64-byte memory word = kMemoryWidthK == kMemoryWidthM
 * (include/MatrixMultiplication.h:18-27 with the default 64-byte bus, CMakeLists.txt:17-19).
 * K and M must be multiples of it (host/RunHardware.cpp:50-61, test/TestSimulation.cpp:22-35). */
MM_API unsigned mm_memory_width(int dtype);

/* hlslib::ocl::Context::Context() (common/OpenCL.h:366-470; host/RunHardware.cpp:116).
 * `device` is the CUDA ordinal (the reference always takes device 0 of the Xilinx platform). */
MM_API int mm_context_create(int device, mm_context **out);
MM_API int mm_context_destroy(mm_context *ctx);

/* Context::MakeBuffer<T, Access>(StorageType, bank, count) (common/OpenCL.h:420-470,502-633;
 * host/RunHardware.cpp:122-138).  Memory banks have no GPU counterpart: one HBM3 pool. */
MM_API int mm_buffer_alloc(mm_context *ctx, size_t bytes, void **device_ptr);
MM_API int mm_buffer_free(mm_context *ctx, void *device_ptr);

/* Buffer::CopyFromHost / Buffer::CopyToHost (common/OpenCL.h:648-720; host/RunHardware.cpp:140-145,
 * 187-190).  Blocking, like the reference. */
MM_API int mm_copy_to_device(mm_context *ctx, void *device_dst, const void *host_src, size_t bytes);
MM_API int mm_copy_to_host(mm_context *ctx, void *host_dst, const void *device_src, size_t bytes);

/* Program::MakeKernel("MatrixMultiplicationKernel", a, b, c, n, k, m) + Kernel::ExecuteTask()
 * (common/OpenCL.h:1346-1379,1486-1504; host/RunHardware.cpp:147-162) on DEVICE buffers.
 * Blocking.  *seconds_device = CUDA-event time around the kernels of this call only (the
 * counterpart of the OpenCL profiling END-START the reference reports); *seconds_wall = host
 * wall clock.  Either may be NULL. */
MM_API int mm_kernel_execute(mm_context *ctx, int dtype, int map_op, int reduce_op, int flags,
                      const void *a_device, const void *b_device, void *c_device, unsigned size_n,
                      unsigned size_k, unsigned size_m, double *seconds_device,
                      double *seconds_wall);

/* Same launch, asynchronous on a caller-supplied CUDA stream (cudaStream_t passed as void*; NULL =
 * the context's own stream), no timing, no synchronisation: for callers that own the stream
 * (benchmark loops, CUDA-graph capture, multi-GPU row-block drivers).  The context's scratch is
 * shared by everything enqueued through it: keep the work of ONE context stream-ordered (one stream
 * at a time) and use one context per concurrently running stream.  Capturable into a CUDA graph
 * once a first call outside capture (or mm_context_reserve) has sized the scratch; see
 * mm_context_reserve for what growth does to captured graphs.  Device pointers must be 16-byte
 * aligned (the reference's buffers are 4096-aligned, include/Utility.h:44-54): MM_ERR_INVALID else. */
MM_API int mm_kernel_enqueue(mm_context *ctx, int dtype, int map_op, int reduce_op, int flags,
                      const void *a_device, const void *b_device, void *c_device, unsigned size_n,
                      unsigned size_k, unsigned size_m, void *cuda_stream);

/* A batch of `batch` same-shape problems in one launch sequence, asynchronous like
 * mm_kernel_enqueue().  Problem i (0 <= i < batch) reads A at a_device + i*N*K elements and B at
 * b_device + i*K*M elements, unless MM_FLAG_BATCH_SHARED_A / _B says every problem reads the first
 * one, and writes C at c_device + i*N*M elements.  Each matrix has the layout of a single call.
 * The result of problem i is BIT-IDENTICAL to mm_kernel_enqueue() on that problem's A and B with the
 * same flags and tuning, for every type, semiring, flag and tuning value.  The call launches the same
 * kernels as one single call (mm_kernel_launch_count()), whatever the batch size: one preparation
 * pass per operand over the whole batch (once for a shared operand) and one compute kernel.
 * Validation as mm_kernel_enqueue(), plus: batch == 0 -> MM_ERR_INVALID; batch > 65535, or
 * batch*N, batch*K or batch*M >= 2^31 -> MM_ERR_UNSUPPORTED.  Scratch grows with the number of
 * distinct operands: size it with mm_context_reserve_batched() before a stream capture. */
MM_API int mm_kernel_enqueue_batched(mm_context *ctx, int dtype, int map_op, int reduce_op, int flags,
                                     const void *a_device, const void *b_device, void *c_device,
                                     unsigned size_n, unsigned size_k, unsigned size_m,
                                     unsigned batch, void *cuda_stream);

/* ---- witnesses: which k each element of a Min / Max product came from ---------------------------
 * mm_kernel_enqueue_witness() computes C exactly as mm_kernel_enqueue_batched() does with the same arguments
 * (BIT-IDENTICAL for every type, map, flag and tuning value, the float default FMNMX included), and beside it
 * W[N x M] (uint32, row-major, packed per problem like C).  W[n,m] is the last k at which the sequential reduction
 * of Naive<> SELECTED its new term t = Map(a[n,k], b[k,m]), with acc the running value:
 *   literal Min `(acc < t) ? acc : t` (every type; float under MM_FLAG_EXACT): selects t when !(acc < t);
 *   literal Max `(t < acc) ? acc : t`: selects t when !(t < acc);
 *     so ties go to the LATEST k, and a NaN term is selected;
 *   FMNMX Min (float without MM_FLAG_EXACT): selects t when t < acc;  FMNMX Max: when acc < t;
 *     so ties go to the EARLIEST k, and a NaN term is never selected;
 * or MM_WITNESS_NONE if no term was ever selected.  Consequences:
 *   - literal path, W != NONE: C has the bits of term W (any NaN payload);
 *   - FMNMX path, W != NONE: C equals term W as a number (C may be -0 where term W is +0, and the reverse, as
 *     documented for MM_FLAG_EXACT);
 *   - W == NONE: C has the bits of the reduce's identity.  A float Max whose terms all lie below FLT_MIN (the
 *     reference's identity numeric_limits<float>::min()) gives NONE, as does an FMNMX Min whose terms all equal FLT_MAX.
 * k counts within the problem: 0 <= W < K whatever the batch index, and with or without MM_FLAG_TRANSPOSED_A.
 * MM_FLAG_BATCH_SHARED_A / _B work as in batched calls; MM_FLAG_TF32X3 is ignored.
 * Validation as mm_kernel_enqueue_batched(), plus: w_device NULL or not 16-byte aligned -> MM_ERR_INVALID;
 * reduce_op other than MM_OP_MIN / MM_OP_MAX -> MM_ERR_INVALID.  W must not overlap A, B or C.  The call uses no
 * scratch, so it can be captured into a CUDA graph without a reserve; per-call profiling records it like a
 * semiring call (no preparation time, the whole call is main time).  Callers detect the feature by this symbol. */
#define MM_WITNESS_NONE 0xFFFFFFFFu
MM_API int mm_kernel_enqueue_witness(mm_context *ctx, int dtype, int map_op, int reduce_op, int flags,
                                     const void *a_device, const void *b_device, void *c_device,
                                     unsigned *w_device, unsigned size_n, unsigned size_k, unsigned size_m,
                                     unsigned batch, void *cuda_stream);

/* ---- accumulation: C <- C (+) (A (x) B) -------------------------------------------------------------
 * mm_kernel_enqueue_accumulate() takes the arguments of mm_kernel_enqueue_batched() and, for problem p and element
 * (n, m), writes
 *     C_new[p,n,m] = R(C_old[p,n,m], P[p,n,m])
 * where P is the value mm_kernel_enqueue_batched() would store there with the same arguments, flags and tuning (bit
 * for bit), and R is ONE application of the reduce operator of the path that computed P, in the data type, with
 * C_old as its FIRST operand:
 *   Add       C_old + P rounded once to nearest-even (float, double, half, bfloat16); integers wrap modulo 2^32
 *             (uint8_t modulo 256).  The tensor-core paths are (Multiply, Add): R is this add on the stored P.
 *   Multiply  C_old * P, likewise
 *   Min       (C_old < P) ? C_old : P      Max  (P < C_old) ? C_old : P
 *             For float without MM_FLAG_EXACT: fminf(C_old, P) / fmaxf(C_old, P) (FMNMX), as the plain call.
 *   And       (C_old != 0 && P != 0) ? 1 : 0
 * The operand order decides the literal Min / Max at ties of +0 and -0 (Min keeps P, Max keeps P) and with NaN (a
 * NaN P is kept; a NaN C_old gives P).  Two consequences of defining the result by P:
 *   - half and bfloat16: P is rounded to 16 bits before the add, so C_new has two roundings (BLAS beta = 1 on a
 *     wider accumulator has one); the reference's Naive<half> rounds after every operation too;
 *   - float Add: C_new is not a sequential reduction seeded with C_old: C (+) (A (x) B) means what its parentheses say.
 * Validation as mm_kernel_enqueue_batched(), in the same order and with the same codes, plus: C (batch*N*M
 * elements) overlapping A ((shared_a ? 1 : batch)*N*K elements) or B ((shared_b ? 1 : batch)*K*M) by one byte ->
 * MM_ERR_INVALID.  A and B may overlap each other; adjacent ranges are accepted.  Path selection, scratch
 * (size it with mm_context_reserve_batched() and the same flags before a stream capture), capture rules,
 * profiling and mm_kernel_launch_count() are those of the batched call.  Device pointers only.  Callers detect the
 * feature by this symbol. */
MM_API int mm_kernel_enqueue_accumulate(mm_context *ctx, int dtype, int map_op, int reduce_op, int flags,
                                        const void *a_device, const void *b_device, void *c_device,
                                        unsigned size_n, unsigned size_k, unsigned size_m,
                                        unsigned batch, void *cuda_stream);

/* ---- closure: all-pairs shortest / longest / widest / most-reliable paths, reachability ------------------------
 * mm_kernel_enqueue_closure() rewrites D in place: `batch` square N x N row-major matrices, packed (problem p starts
 * at d_device + p*N*N elements), by blocked Floyd–Warshall over (Map, R), R = reduce_op = MM_OP_MIN or MM_OP_MAX.
 * Asynchronous like the other enqueue entries.  It does NOT initialise the diagonal: callers who want reflexive paths
 * set D[i][i] to the Map's identity themselves (0 for min-plus).
 *
 * b = mm_closure_block(dtype) = 128 for every type (the semiring kernels' CTA tile).  Blocks K_r = [r*b, min((r+1)*b,
 * N)); the last may be partial, with a width that is a multiple of the memory width.  A "step k" updates its set of
 * (i, j) simultaneously, every read of the step seeing the values from before it:
 *     D'[i][j] = R(D[i][j], Map(D[i][k], D[k][j]))
 * Round r = 0, 1, ... has three phases:
 *   1. diagonal:  for k in K_r ascending, step k over i, j in K_r;
 *   2. panels:    for k in K_r ascending, step k over i in K_r, j not in K_r (row panel) and over i not in K_r,
 *                 j in K_r (column panel); the two panels are independent given phase 1;
 *   3. remainder: for i, j not in K_r, D[i][j] <- R(...R(R(D[i][j], t_k0), t_k0+1)..., t_klast), t_k =
 *                 Map(D[i][k], D[k][j]), the k running over K_r ascending, the panels as phase 2 left them, and the
 *                 accumulator SEEDED WITH D[i][j], never with the reduce's identity (a float (Multiply, Max)
 *                 reliability matrix keeps its "no path" zeros; the plain product would seed with FLT_MIN).
 * Map and R are the functors of the product, one rounding each: float at flags 0 uses fminf / fmaxf (FMNMX) for Min /
 * Max, under MM_FLAG_EXACT the literal (a < b) ? a : b, as mm_kernel_enqueue() does.  Consequences:
 *   - with exact arithmetic the result is the true closure whatever b is: integers without wrap, Min / Max / And
 *     maps, and float or double data whose path sums are exact;
 *   - with rounding Add / Multiply maps, each element is a path weight rounded in the order stated above;
 *   - integer Add wraps modulo 2^32 (uint8_t modulo 256) exactly as in the product, so INT_MAX as "no edge" is the
 *     caller's to avoid (use a bound whose sums do not wrap);
 *   - a negative (improving) cycle gives whatever the definition gives; the caller detects it on the diagonal.
 * Validation as mm_kernel_enqueue_witness() with K = M = N, in the same order and with the same codes (N % the memory
 * width != 0 -> MM_ERR_SHAPE; batch and extent limits of the batched call), plus: reduce_op other than MM_OP_MIN /
 * MM_OP_MAX -> MM_ERR_INVALID; MM_FLAG_TRANSPOSED_A, MM_FLAG_BATCH_SHARED_A or _B -> MM_ERR_INVALID.
 * MM_FLAG_TF32X3 is ignored.  The call uses no scratch, so it can be captured into a CUDA graph without a reserve;
 * per-call profiling records it like a semiring call (the whole call is main time).  It launches 3 kernels per block
 * of indices (1 when N <= b). */
MM_API int mm_kernel_enqueue_closure(mm_context *ctx, int dtype, int map_op, int reduce_op, int flags,
                                     void *d_device, unsigned size_n, unsigned batch, void *cuda_stream);
/* b of mm_kernel_enqueue_closure() for `dtype`; 0 for an unknown dtype. */
MM_API unsigned mm_closure_block(int dtype);

/* ---- bit-packed Boolean matrices: products and transitive closure on the b1 tensor cores -----------------------
 * Layout: an R x L Boolean matrix is stored bit-packed and row-major, element (i, j) = bit j % 8 (least significant
 * first) of byte i*L/8 + j/8, i.e. numpy.packbits(X, axis=-1, bitorder='little').  A batch is packed: problem p starts
 * at byte p*R*L/8.  Every offset is 64-bit.
 *
 * mm_kernel_enqueue_bool(): C[p][i][j] = 1 iff some k has A[p][i][k] = B[p][k][j] = 1, for A N x K, B K x M (row-major)
 * and C N x M, on wgmma m64nNk256 .b1.and.popc: exact counts of A AND B, stored as count > 0.  Asynchronous like the
 * other enqueue entries; every bit of C is written (with M a multiple of 128, rows of C have no padding bits).  It
 * keeps a K-major copy of B (batch*K*M/8 bytes) in the context's scratch, sized by a first call outside a stream
 * capture; per-call profiling records that copy as preparation and the product as main time.  The wgmma tuning knobs
 * apply (cta_group, block_n, stages, raster_rows, tile_sync, tma_store, l2_policy) and give the same bits.
 *
 * mm_kernel_enqueue_bool_closure(): `batch` packed N x N matrices D become D+ in place: D+[i][j] = 1 iff a path of one
 * or more edges leads from i to j.  The diagonal is 1 exactly where i lies on a cycle (self-loops included): the call
 * does not set the reflexive diagonal, as mm_kernel_enqueue_closure() does not initialise it.  The result is
 * BIT-IDENTICAL to mm_kernel_enqueue_closure(MM_DTYPE_UINT8, MM_OP_AND, MM_OP_MAX, 0, ...) on the unpacked 0/1 bytes,
 * after packing.  Blocked Floyd–Warshall; the block size cannot be observed in the result.  No scratch: it can be
 * captured into a CUDA graph without a prior call.  Per-call profiling records the whole call as main time.
 *
 * Validation, in this order: null context or pointer, or N, K or M equal to 0 -> MM_ERR_INVALID; K or M (closure: N)
 * not a multiple of 128 -> MM_ERR_SHAPE; the batch limits of mm_kernel_enqueue_batched(); pointers not 16-byte aligned
 * -> MM_ERR_INVALID; flags != 0 (reserved) -> MM_ERR_INVALID; product: C's bytes overlapping A's or B's ->
 * MM_ERR_INVALID.  mm_kernel_launch_count(), mm_kernel_path() and the tuning enum do not describe these calls.
 * Callers detect the feature by these symbols. */
MM_API int mm_kernel_enqueue_bool(mm_context *ctx, int flags, const void *a_device, const void *b_device,
                                  void *c_device, unsigned size_n, unsigned size_k, unsigned size_m,
                                  unsigned batch, void *cuda_stream);
MM_API int mm_kernel_enqueue_bool_closure(mm_context *ctx, int flags, void *d_device, unsigned size_n,
                                          unsigned batch, void *cuda_stream);

/* Per-phase device timing of enqueued work, for roofline accounting.  With profiling on, every
 * mm_kernel_enqueue()/mm_kernel_execute() records CUDA events on the launching stream around
 * (i) the operand-preparation kernels and (ii) the main compute kernel.  mm_context_profile_read()
 * synchronises on the recorded events, returns the SUMS over the calls since the last read (at
 * most 256 calls are kept) and the number of calls, and resets the counters. */
MM_API int mm_context_set_profiling(mm_context *ctx, int enable);
MM_API int mm_context_profile_read(mm_context *ctx, double *prep_seconds_sum,
                                   double *main_seconds_sum, int *calls);

/* Number of kernels one mm_kernel_enqueue() with these arguments launches (for accounting). */
MM_API int mm_kernel_launch_count(int dtype, int map_op, int reduce_op, int flags);

/* Name of the compute kernel family mm_kernel_enqueue() would dispatch to for a small problem
 * ("wgmma_tf32", "wgmma_f16", "wgmma_bf16", "wgmma_i8", "dmma_f64", "semiring_simt"); static string. */
MM_API const char *mm_kernel_path(int dtype, int map_op, int reduce_op, int flags);

/* The reference's simulation entry, extern "C" MatrixMultiplicationKernel(a, b, c, n, k, m)
 * (include/MatrixMultiplication.h:155-171, called with HOST pointers at
 * test/TestSimulation.cpp:66), for a run-time chosen configuration: host -> device copies,
 * the kernel, device -> host copy of C; blocking.  With `ctx` NULL it uses (and lazily creates) a
 * per-process default: one context on device $MM_DEVICE (default 0), or — when the environment
 * variable MM_NUM_GPUS is G > 1 and A is row-major — an mm_multi over devices 0..G-1, i.e. the
 * call is split over G GPUs exactly like mm_multi_gemm_host().  Timings optional as above;
 * *seconds_device covers the kernels only. */
MM_API int mm_gemm_host(mm_context *ctx, int dtype, int map_op, int reduce_op, int flags,
                 const void *a_host, const void *b_host, void *c_host, unsigned size_n,
                 unsigned size_k, unsigned size_m, double *seconds_device, double *seconds_wall);

/* ---- tuning -------------------------------------------------------------------------------------
 * Run-time counterpart of the reference's configure-time tile / parallelism knobs
 * (CMakeLists.txt:17-29: MM_PARALLELISM_*, MM_MEMORY_TILE_SIZE_*), which scripts/build_manager.py:224-306
 * sweeps by rebuilding.  Here every variant is compiled into the library and selected per context.
 * Defaults are the measured best; the environment variable named with each knob, read ONCE at
 * mm_context_create(), overrides the default; mm_context_set_tuning() overrides both.  Every value
 * computes the same C (the parity suite runs under each). */
enum {
  MM_TUNE_TCGEN05_CTA_GROUP = 0,   /* 1 | 2: single-CTA tiles or 2-CTA clusters sharing B (default 2)  MM_TCGEN05_CTA_GROUP */
  MM_TUNE_TCGEN05_BLOCK_N = 1,     /* 128 | 256: C tile columns = wgmma N (default 256)                MM_TCGEN05_BLOCK_N */
  MM_TUNE_TCGEN05_STAGES = 2,      /* TMA ring depth, 0 = deepest that fits (default), else 2..8       MM_TCGEN05_STAGES */
  MM_TUNE_TCGEN05_RASTER_ROWS = 3, /* C rows per rasterisation group = L2 "memory tile" height (2048)  MM_TCGEN05_RASTER_ROWS */
  MM_TUNE_TCGEN05_TILE_SYNC = 4,   /* 0 | 1: soft wave barrier between co-running tiles (default 1)    MM_TCGEN05_TILE_SYNC */
  MM_TUNE_TCGEN05_B_MN = 5,        /* 0 | 1: accepted, no effect on sm_90a: wgmma reads tf32 and 8-bit
                                      operands only K-major, so B is always a transposed copy         MM_TCGEN05_B_MN */
  MM_TUNE_TCGEN05_L2_POLICY = 6,   /* TMA loads' L2 eviction priority: 0 normal, 1 first, 2 last       MM_TCGEN05_L2 */
  MM_TUNE_TCGEN05_B_OVERLAP = 7,   /* 0 | 1: accepted, no effect on sm_90a: B's preparation always
                                      completes before the GEMM starts                               MM_TCGEN05_B_OVERLAP */
  MM_TUNE_TCGEN05_TMA_STORE = 8,   /* 0 | 1: epilogue through shared memory + TMA stores (default 1)   MM_TCGEN05_TMA_STORE */
  MM_TUNE_DMMA_TILE_ROWS = 9,      /* 0 = automatic | 64 | 128: CTA tile rows of the double kernel     MM_DMMA_TILE_ROWS */
  MM_TUNE_EXPERIMENT_TF32_NO_ROUND = 10, /* 1: feed raw fp32 bits to tf32 wgmma (measures the truncation
                                      bias that motivates the rounding pass; never for production)    MM_EXPERIMENT_TF32_NO_ROUND */
  MM_TUNE_SEMIRING_RING = 11,      /* 0 | 1: CUDA-core kernel for 4-byte types with both tiles in a TMA ring and no
                                      block-wide barrier (default 1), or the register-staged kernel       MM_SEMIRING_RING */
  MM_TUNE_COUNT = 12
};
MM_API int mm_context_set_tuning(mm_context *ctx, int knob, int value);
MM_API int mm_context_get_tuning(mm_context *ctx, int knob, int *value);

/* Pre-size the context's scratch for the largest problem that will be enqueued.  The scratch grows
 * on demand otherwise; growth reallocates it, which INVALIDATES any CUDA graph captured through
 * mm_kernel_enqueue() earlier (the old scratch addresses are baked into the graph).  A context that
 * has seen a stream capture therefore keeps superseded allocations alive until it is destroyed. */
MM_API int mm_context_reserve(mm_context *ctx, int dtype, int flags, unsigned size_n, unsigned size_k,
                              unsigned size_m);
/* The same for mm_kernel_enqueue_batched() with these flags: one operand copy per problem, or one
 * for an operand the flags mark as shared.  Batch rules as mm_kernel_enqueue_batched(). */
MM_API int mm_context_reserve_batched(mm_context *ctx, int dtype, int flags, unsigned size_n,
                                      unsigned size_k, unsigned size_m, unsigned batch);

/* ---- multi-GPU: C row-blocks over the GPUs of one box (SURVEY.md section 8e) ------------------
 * The reference's API is ONE blocking call on host pointers (include/MatrixMultiplication.h:155-171)
 * and one device-resident lifecycle (host/RunHardware.cpp:116-190); outer tiles of C are independent
 * (kernel/Compute.cpp:53-56).  mm_multi keeps both shapes over G devices of this process: GPU g owns
 * rows [g*ceil(N/G), ...) of A and C; every GPU uploads only ITS 1/G row-slice of B over PCIe and the
 * slices are all-gathered GPU-to-GPU over NVLink into each device's B by the library's own kernel
 * reading peer memory, on every path; each device then prepares its B locally.  No collective per
 * step, no reduction (K is not split).  All fan-out is internal (one host thread per GPU) and joined
 * before the call returns.
 * A stored K x N (MM_FLAG_TRANSPOSED_A) cannot be cut into contiguous row blocks: MM_ERR_UNSUPPORTED. */
typedef struct mm_multi mm_multi;
/* `devices` = n_gpus CUDA ordinals, or NULL for 0 .. n_gpus-1. */
MM_API int mm_multi_create(int n_gpus, const int *devices, mm_multi **out);
MM_API int mm_multi_destroy(mm_multi *multi);
MM_API int mm_multi_device_count(const mm_multi *multi);
/* The per-device context (for mm_context_set_tuning); owned by `multi`. */
MM_API mm_context *mm_multi_context(mm_multi *multi, int index);
/* How an N x K x M problem is cut over `n_gpus` devices — pure arithmetic, no device needed; the same rule every
 * mm_multi_* entry applies.  GPU `index` owns rows [*row_begin, *row_end) of A and C (ceil(N / G) rows each, tail GPUs
 * may own fewer or none) and uploads the K-rows [*b_row_begin, *b_row_end) of B (slices of ceil(K / G) rounded up to
 * a multiple of 64 rows; the whole of B when there is no peer access).  Callers use it to place their host matrices
 * (e.g. each block on the NUMA node of the GPU that copies it).  Any output pointer may be NULL. */
MM_API int mm_multi_partition(int n_gpus, int index, unsigned size_n, unsigned size_k, unsigned *row_begin,
                              unsigned *row_end, unsigned *b_row_begin, unsigned *b_row_end);
/* 1 if every pair of devices has peer access (NVLink gather), 0 if B falls back to a full upload per GPU. */
MM_API int mm_multi_peer_access(const mm_multi *multi);
/* MatrixMultiplicationKernel(a, b, c, n, k, m) with HOST pointers over all G devices; blocking.
 * *seconds_device = the slowest GPU's first-kernel-start .. last-kernel-end. */
MM_API int mm_multi_gemm_host(mm_multi *multi, int dtype, int map_op, int reduce_op, int flags,
                              const void *a_host, const void *b_host, void *c_host, unsigned size_n,
                              unsigned size_k, unsigned size_m, double *seconds_device,
                              double *seconds_wall);
/* Device-resident lifecycle, the multi-GPU form of MakeBuffer + CopyFromHost / ExecuteTask / CopyToHost
 * (host/RunHardware.cpp:122-190): upload = A row-blocks + B slices over PCIe, B assembled on every
 * GPU over NVLink; execute = the kernels of every GPU on the resident buffers (device seconds = the
 * slowest GPU's CUDA-event time around its kernels); download = C row-blocks to the host.
 * The resident operands live in the same per-device staging buffers that mm_multi_gemm_host() and mm_gemm_host()
 * on a member context (mm_multi_context()) use.  Execute and download therefore return MM_ERR_INVALID, never
 * MM_OK over other operands, unless the last upload on this multi succeeded, had the same type and sizes, and no
 * call has reused any member context's staging buffers since.  Download also needs an execute after that upload.
 * (Since version 203; earlier versions computed on, or returned, whatever those buffers held.) */
MM_API int mm_multi_upload(mm_multi *multi, int dtype, int flags, const void *a_host, const void *b_host,
                           unsigned size_n, unsigned size_k, unsigned size_m);
MM_API int mm_multi_execute(mm_multi *multi, int dtype, int map_op, int reduce_op, int flags,
                            unsigned size_n, unsigned size_k, unsigned size_m, double *seconds_device,
                            double *seconds_wall);
MM_API int mm_multi_download(mm_multi *multi, int dtype, void *c_host, unsigned size_n, unsigned size_m);

/* Library/ABI version (major * 100 + minor). */
MM_API int mm_version(void);

#ifdef __cplusplus
}
#endif

#endif /* MM_B200_H_ */
