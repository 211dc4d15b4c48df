// Shared host-side helpers for the CUDA translation units of libmm_b200.so.
#pragma once

#include <cuda_runtime.h>

#include <cstdio>
#include <functional>
#include <string>

#include "../../include/mm_b200.h"

namespace mm {

// Multi-GPU calls (capi.cu): called by each device's float GEMM path once its rows of A are prepared and before
// its first GEMM, with its fits word of A (HalfScratch::fits_a, or null without fp16 copies) and the stream that
// prepared it.  It returns once every device has called it, with the word cleared unless the whole A fits.
using AgreeFn = std::function<int(unsigned int *fits_a, cudaStream_t stream)>;

// Thread-local error message behind mm_last_error().
void set_error(const std::string &msg);
int fail(int code, const std::string &msg);

#define MM_CUDA_TRY(expr)                                                                  \
  do {                                                                                     \
    cudaError_t err__ = (expr);                                                            \
    if (err__ != cudaSuccess) {                                                            \
      return ::mm::fail(MM_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(err__)); \
    }                                                                                      \
  } while (0)

inline unsigned ceil_div(unsigned a, unsigned b) { return (a + b - 1) / b; }

// Scratch the tensor-core path needs (rounded / transposed operand copies); owned by the
// context, grown on demand, reused across calls.
struct Scratch {
  void *ptr = nullptr;
  size_t bytes = 0;
};

// Run-time tuning of the kernel families: the GPU counterpart of the reference's CMake-time tile /
// parallelism knobs (CMakeLists.txt:17-29), selected at run time where
// scripts/build_manager.py:224-306 rebuilds.  One instance per context: defaults, then the
// MM_TUNE_* environment variables read ONCE at mm_context_create(), then mm_context_set_tuning().
// Indexed by the MM_TUNE_* codes of include/mm_b200.h.
struct Tuning {
  int v[MM_TUNE_COUNT];
  int cta_group() const { return v[MM_TUNE_TCGEN05_CTA_GROUP]; }
  int block_n() const { return v[MM_TUNE_TCGEN05_BLOCK_N]; }
  int stages() const { return v[MM_TUNE_TCGEN05_STAGES]; }
  int raster_rows() const { return v[MM_TUNE_TCGEN05_RASTER_ROWS]; }
  bool tile_sync() const { return v[MM_TUNE_TCGEN05_TILE_SYNC] != 0; }
  int l2_policy() const { return v[MM_TUNE_TCGEN05_L2_POLICY]; }
  bool tma_store() const { return v[MM_TUNE_TCGEN05_TMA_STORE] != 0; }
  int dmma_tile_rows() const { return v[MM_TUNE_DMMA_TILE_ROWS]; }
  bool tf32_no_round() const { return v[MM_TUNE_EXPERIMENT_TF32_NO_ROUND] != 0; }
  bool semiring_ring() const { return v[MM_TUNE_SEMIRING_RING] != 0; }
};
Tuning default_tuning();                                  // capi.cu
int tuning_validate(int knob, int value);                 // MM_OK or MM_ERR_INVALID (message set)

// A batch of `count` same-shape problems (mm_kernel_enqueue_batched).  Problem i reads A at
// a + i * N * K elements and B at b + i * K * M, unless the operand is shared (every problem reads
// the first one), and writes C at c + i * N * M.  A single call is a batch of one.
struct GemmBatch {
  unsigned count = 1;
  bool shared_a = false, shared_b = false;
  unsigned a_copies() const { return shared_a ? 1u : count; }  // distinct A (B) operands of the batch
  unsigned b_copies() const { return shared_b ? 1u : count; }
};

struct GemmArgs {
  const void *a;
  const void *b;
  void *c;
  unsigned n, k, m;
  int flags;
  cudaStream_t stream;
  const Tuning *tuning = nullptr;  // never null on a real launch (capi.cu fills it from the context)
  GemmBatch batch;
  // optional profiling event (capi.cu): recorded by the launcher between operand preparation
  // and the main kernel when non-null
  cudaEvent_t ev_prep_done = nullptr;
  // Resource-preparation pass: do everything a launch does EXCEPT enqueue kernels (set function
  // attributes, which also forces the lazily loaded cubin in).  mm_kernel_execute runs it before
  // recording its start event so that the reported device time is kernel time only.
  bool dry_run = false;
  // mm_kernel_enqueue_accumulate: C <- Reduce(C_old, product), C_old read in the compute kernel's epilogue
  bool accumulate = false;
  // mm_multi_execute: the devices' agreement on the datapath of the whole A (AgreeFn), or null
  const AgreeFn *agree = nullptr;
};

// ---- kernel families (one launcher per translation unit) ---------------------------------------
// CUDA-core semiring tile kernel, any (dtype, map, reduce).  semiring_*.cu
int launch_semiring(int dtype, int map_op, int reduce_op, const GemmArgs &args);
// The same C for a Min / Max reduce, plus the witness W (N x M uint32 per problem).  semiring_witness_*.cu
int launch_semiring_witness(int dtype, int map_op, int reduce_op, const GemmArgs &args, unsigned *w);
// C <- Reduce(C_old, product) with the same kernel choice as launch_semiring.  semiring_accumulate_*.cu
int launch_semiring_accumulate(int dtype, int map_op, int reduce_op, const GemmArgs &args);
// Closure of `batch` packed N x N problems at d in place over a Min / Max reduce (mm_kernel_enqueue_closure), by
// blocked Floyd–Warshall; float Min / Max take FMNMX unless MM_FLAG_EXACT.  semiring_closure_*.cu
int launch_semiring_closure(int dtype, int map_op, int reduce_op, int flags, void *d, unsigned n, unsigned batch,
                            cudaStream_t stream);

// wgmma tensor-core GEMM for (Multiply, Add) float (tf32), half (f16) and uint8_t (u8).
// The context's scratch holds, in this order: [B operand copy][B fp16][A operand copy][A fp16] ... [fits][wave-barrier counter].
//   B operand copy: the transposed M x K copy wgmma reads K-major, rounded to TF32 for float.
//   A operand copy: float = A rounded to TF32; any type with MM_FLAG_TRANSPOSED_A = A transposed.
//   fp16 copies and fits flags (float on the default TF32 datapath only, see HalfScratch): the rounded copies again as
//   halves, and per distinct operand whether every value of it is exactly a half.
// A batch keeps one copy per distinct operand (GemmBatch::a_copies / b_copies), packed.
size_t tcgen05_scratch_bytes(int dtype, unsigned n, unsigned k, unsigned m, int flags, const Tuning &t,
                             const GemmBatch &batch = GemmBatch{});
size_t tcgen05_bt_bytes(int dtype, unsigned k, unsigned m, int flags, const Tuning &t,
                        unsigned b_copies = 1);  // = offset of the A copy
int launch_tcgen05(int dtype, const GemmArgs &args, void *scratch, size_t scratch_bytes);
// Float's fp16 operand copies and their fits flags as the GEMM reads them: a problem whose A and B both fit runs on
// the f16 wgmma.  All null: TF32 only.
struct HalfOperands {
  const void *a = nullptr, *b = nullptr;
  const unsigned int *fits_a = nullptr, *fits_b = nullptr;
};
// Where the preparation writes them.  Just before the wave-barrier counter at the scratch's end: [one fits word per B copy][one per
// A copy][pending map of B][pending map of A], all set nonzero by one cudaMemsetAsync of flag_bytes before the
// preparation.  A fits word is cleared by any preparation item that meets a value which is not exactly a normal half or
// zero (fits_half.h).  The pending maps hold one byte per 64 x 64 item of each copy: 1 while the item's TF32 copy is
// owed (tcgen05_prepare_float).  All null when the call stays on TF32: not float, MM_FLAG_TF32X3 (its lo parts are far
// below half range) or the tf32_no_round experiment (raw float bits).
struct HalfScratch {
  void *a = nullptr, *b = nullptr;
  unsigned int *fits_a = nullptr, *fits_b = nullptr;
  unsigned char *pending_a = nullptr, *pending_b = nullptr;
  size_t flag_bytes = 0;
  HalfOperands operands() const { return HalfOperands{a, b, fits_a, fits_b}; }
};
HalfScratch tcgen05_half_scratch(void *scratch, size_t scratch_bytes, int dtype, unsigned n, unsigned k, unsigned m,
                                 int flags, const Tuning &t, const GemmBatch &batch = GemmBatch{});
// The phases of launch_tcgen05, for callers that reuse a prepared B across row-blocks (the pipelined
// host path, the multi-GPU row-block driver).
// The soft wave-barrier counter of the GEMM, at the tail of the scratch (zeroed by the launcher before use).
unsigned int *tcgen05_tile_sync(void *scratch, size_t scratch_bytes);
// The K-major copy of B (M x K, one K x M array `b` per copy) into `bt` on `stream`: the hi / lo split for
// MM_FLAG_TF32X3, the unrounded transpose for float under the tf32_no_round experiment, the transpose for half,
// bfloat16 and uint8_t.  *b_op receives the kernel's B operand (bt).  `copies` packed K x M problems of B are prepared
// into `copies` packed M x K copies.  Not for float on the default datapath: see tcgen05_prepare_float.
int tcgen05_prepare_b(int dtype, const void *b, void *bt, unsigned k, unsigned m, int flags, const Tuning &t,
                      const void **b_op, cudaStream_t stream, unsigned copies = 1);
// `copies` packed problems of `rows` rows each.  Not for float on the default datapath: see tcgen05_prepare_float.
int tcgen05_prepare_a(int dtype, const void *a, void *aprep, unsigned rows, unsigned k, int flags, const Tuning &t,
                      const void **a_op, cudaStream_t stream, unsigned copies = 1);
// Float on the default datapath (HalfScratch non-empty): both operands into the scratch's copies, the TF32 copy (B^T
// at the scratch's start, A at tcgen05_bt_bytes) or the fp16 copy of each 64 x 64 item, whichever the GEMM will read.
// Needs the memset of HalfScratch::flag_bytes first.  complete = false: the first pass over B (`b` non-null, one K x M
// array per copy) and rows [row0, row0 + rows) of A (`a` non-null, pointing at row row0; row0 % 64 == 0; A stored
// K x N only whole); it may run per chunk of A.  complete = true, once the fits words are final (after any multi-GPU
// agreement): the second pass over the whole of both, which writes the TF32 copies still owed.  One launch each.
int tcgen05_prepare_float(bool complete, const void *a, unsigned row0, unsigned rows, const void *b, unsigned n,
                          unsigned k, unsigned m, int flags, const Tuning &t, const GemmBatch &batch, void *scratch,
                          size_t scratch_bytes, cudaStream_t stream);
// `tile_sync`: device counter for the kernel's soft wave barrier, or null.
int tcgen05_gemm(int dtype, const void *a_op, const void *b_op, void *c, unsigned rows, unsigned k, unsigned m,
                 int flags, const Tuning &t, unsigned int *tile_sync, cudaStream_t stream,
                 const GemmBatch &batch = GemmBatch{}, bool accumulate = false,
                 const HalfOperands &half = HalfOperands{});
constexpr size_t kTcgen05TailBytes = 256;  // [wave-barrier counter, 256 B]
// The NVLink all-gather of the multi-GPU path, for every kernel family: row-sliced B into one local K x M array
// `dst`.  K-row r is read through parts[r / part_rows], a DEVICE array of pointers to FULL-size K x M arrays (the
// devices' B buffers) of which only that slice's rows need to be valid; rows already in `dst` are not copied.
int gather_b_rows(const void *const *parts, unsigned part_rows, void *dst, size_t elem_bytes, unsigned k, unsigned m,
                  cudaStream_t stream);

// Bit-packed Boolean matrices (mm_kernel_enqueue_bool / _closure); every offset in bytes, rows of (columns / 8) bytes.
// `batch` packed K x M bit matrices at b -> their M x K transposes at bt.  gemm_wgmma_b1.cu
int bool_transpose_b(const void *b, void *bt, unsigned k, unsigned m, unsigned batch, cudaStream_t stream);
// C[N x M] = A[N x K] . B'^T on the b1 wgmma, B' the M x K copy of bool_transpose_b.  gemm_wgmma_b1.cu
int bool_gemm(const void *a, const void *bt, void *c, unsigned n, unsigned k, unsigned m, unsigned batch,
              const Tuning &t, unsigned int *tile_sync, cudaStream_t stream);
// `batch` packed N x N bit matrices at d -> their transitive closures, in place.  bool_closure.cu
int bool_closure(void *d, unsigned n, unsigned batch, cudaStream_t stream);

// DMMA (mma.sync m8n8k4 f64) GEMM for (Multiply, Add) double.  gemm_dmma.cu
int launch_dmma(const GemmArgs &args);
// The same with C <- C_old + product.  gemm_dmma_acc.cu
int launch_dmma_accumulate(const GemmArgs &args);

}  // namespace mm
