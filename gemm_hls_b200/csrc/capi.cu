// C-ABI of libmm_b200.so (include/mm_b200.h): context / buffer lifecycle mirroring the
// hlslib::ocl calls of host/RunHardware.cpp:116-190, the dispatch of one
// MatrixMultiplicationKernel invocation onto the sm_90a kernel families, the pipelined host-pointer
// entry (test/TestSimulation.cpp:66) and its row-block split over the GPUs of one box.
#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "common.cuh"

namespace mm {

namespace {
thread_local std::string g_last_error = "";
}

void set_error(const std::string &msg) { g_last_error = msg; }
int fail(int code, const std::string &msg) {
  set_error(msg);
  return code;
}

namespace {

struct KnobInfo {
  const char *env;
  int dflt;
};
// index = MM_TUNE_* (include/mm_b200.h)
const KnobInfo kKnobs[MM_TUNE_COUNT] = {
    {"MM_TCGEN05_CTA_GROUP", 2}, {"MM_TCGEN05_BLOCK_N", 256},  {"MM_TCGEN05_STAGES", 0},
    {"MM_TCGEN05_RASTER_ROWS", 2048}, {"MM_TCGEN05_TILE_SYNC", 1}, {"MM_TCGEN05_B_MN", 1},
    {"MM_TCGEN05_L2", 0}, {"MM_TCGEN05_B_OVERLAP", 0}, {"MM_TCGEN05_TMA_STORE", 1},
    {"MM_DMMA_TILE_ROWS", 0}, {"MM_EXPERIMENT_TF32_NO_ROUND", 0}, {"MM_SEMIRING_RING", 1},
};

}  // namespace

int tuning_validate(int knob, int value) {
  bool ok = false;
  switch (knob) {
    case MM_TUNE_TCGEN05_CTA_GROUP: ok = value == 1 || value == 2; break;
    case MM_TUNE_TCGEN05_BLOCK_N: ok = value == 128 || value == 256; break;
    case MM_TUNE_TCGEN05_STAGES: ok = value == 0 || (value >= 2 && value <= 8); break;
    case MM_TUNE_TCGEN05_RASTER_ROWS: ok = value >= 1; break;
    case MM_TUNE_TCGEN05_L2_POLICY: ok = value >= 0 && value <= 2; break;
    case MM_TUNE_DMMA_TILE_ROWS: ok = value == 0 || value == 64 || value == 128; break;
    case MM_TUNE_TCGEN05_TILE_SYNC:
    case MM_TUNE_TCGEN05_B_MN:
    case MM_TUNE_TCGEN05_B_OVERLAP:
    case MM_TUNE_TCGEN05_TMA_STORE:
    case MM_TUNE_EXPERIMENT_TF32_NO_ROUND:
    case MM_TUNE_SEMIRING_RING: ok = value == 0 || value == 1; break;
    default: return fail(MM_ERR_INVALID, "unknown tuning knob " + std::to_string(knob));
  }
  if (!ok) {
    return fail(MM_ERR_INVALID, std::string("value ") + std::to_string(value) + " is out of range for tuning knob " +
                                    kKnobs[knob].env);
  }
  return MM_OK;
}

Tuning default_tuning() {
  Tuning t;
  for (int i = 0; i < MM_TUNE_COUNT; ++i) {
    t.v[i] = kKnobs[i].dflt;
    const char *e = std::getenv(kKnobs[i].env);
    if (!e || !*e) continue;
    int value;
    if (i == MM_TUNE_TCGEN05_L2_POLICY && (e[0] == 'n' || e[0] == 'f' || e[0] == 'l')) {
      value = e[0] == 'f' ? 1 : (e[0] == 'l' ? 2 : 0);  // normal / first / last, as the round-1 scripts spell it
    } else {
      value = std::atoi(e);
    }
    if (tuning_validate(i, value) == MM_OK) t.v[i] = value;  // an out-of-range environment value is ignored
  }
  return t;
}

}  // namespace mm

struct mm_context {
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaStream_t copy_in = nullptr, copy_out = nullptr;  // H2D / D2H streams of the pipelined host path
  std::vector<cudaEvent_t> sync_events;                // untimed events ordering the streams
  cudaEvent_t ev_start = nullptr, ev_stop = nullptr;
  cudaEvent_t ev_slice = nullptr;                      // multi-GPU: this device's slice of B has arrived
  mm::Scratch scratch;       // operand copies of the tensor-core path
  mm::Scratch staging[3];    // device A, B, C of the host-pointer entries
  uint64_t staging_gen = 0;  // bumped by every call that writes staging[]: mm_multi_* checks its upload is still there
  std::vector<void *> retired;  // superseded scratch allocations a captured graph may still reference
  bool captured = false;        // a stream capture has gone through this context
  mm::Tuning tuning;
  bool profiling = false;
  std::vector<cudaEvent_t> prof_events;  // 3 per profiled call: start, after prep, after main
  int prof_calls = 0;
  std::mutex mutex;          // entry points are blocking and serialised per context, like
                             // hlslib::ocl::Context's enqueue/memcopy mutexes (common/OpenCL.h:474-492)
};

namespace {

using mm::fail;

bool valid_dtype(int d) { return d >= 0 && d < MM_DTYPE_COUNT; }
bool valid_op(int o) { return o >= 0 && o < MM_OP_COUNT; }

enum Path { kPathTcgen05, kPathDmma, kPathSemiring };

// The types the wgmma GEMM takes for (Multiply, Add).
bool tensor_core_dtype(int d) {
  return d == MM_DTYPE_FLOAT || d == MM_DTYPE_HALF || d == MM_DTYPE_BFLOAT16 || d == MM_DTYPE_UINT8;
}

// uint8_t on the integer tensor cores: products accumulate exactly in 32-bit integers while 255^2 * K < 2^31; the low byte
// of the exact sum is the reference's modulo-256 arithmetic.  Longer K takes the CUDA-core kernel.
constexpr unsigned kMaxKInt8Tensor = 33024;

Path select_path(int dtype, int map_op, int reduce_op, int flags, unsigned n, unsigned k) {
  const bool dense = (map_op == MM_OP_MULTIPLY && reduce_op == MM_OP_ADD) && !(flags & MM_FLAG_EXACT);
  if (dense && (dtype == MM_DTYPE_FLOAT || dtype == MM_DTYPE_HALF || dtype == MM_DTYPE_BFLOAT16)) return kPathTcgen05;
  if (dense && dtype == MM_DTYPE_UINT8 && k <= kMaxKInt8Tensor) return kPathTcgen05;
  if (dense && dtype == MM_DTYPE_DOUBLE) {
    // the DMMA kernel reads a transposed A through 16-byte boxes: needs an even N
    return ((flags & MM_FLAG_TRANSPOSED_A) && (n % 2 != 0)) ? kPathSemiring : kPathDmma;
  }
  return kPathSemiring;
}

// Grow `s` to at least `bytes`.  `keep_old`: the superseded allocation stays alive (a captured CUDA
// graph may hold its address) and is freed with the context.
int ensure(mm_context *ctx, mm::Scratch &s, size_t bytes, bool keep_old) {
  if (s.bytes >= bytes) return MM_OK;
  if (s.ptr) {
    if (keep_old) ctx->retired.push_back(s.ptr);
    else cudaFree(s.ptr);
  }
  s.ptr = nullptr;
  s.bytes = 0;
  cudaError_t e = cudaMalloc(&s.ptr, bytes);
  if (e != cudaSuccess) {
    return fail(e == cudaErrorMemoryAllocation ? MM_ERR_NOMEM : MM_ERR_CUDA,
                std::string("cudaMalloc(") + std::to_string(bytes) + "): " + cudaGetErrorString(e));
  }
  s.bytes = bytes;
  return MM_OK;
}

int check_args(int dtype, int map_op, int reduce_op, const void *a, const void *b, const void *c,
               unsigned n, unsigned k, unsigned m) {
  if (!valid_dtype(dtype)) return fail(MM_ERR_INVALID, "unknown MM_DATA_TYPE code");
  if (!valid_op(map_op) || !valid_op(reduce_op)) return fail(MM_ERR_INVALID, "unknown MM_MAP_OP / MM_REDUCE_OP code");
  if (!a || !b || !c) return fail(MM_ERR_INVALID, "null matrix pointer");
  if (n == 0 || k == 0 || m == 0) return fail(MM_ERR_INVALID, "matrix dimensions must be positive");
  const unsigned w = mm_memory_width(dtype);
  // same rule and wording as host/RunHardware.cpp:50-61
  if (k % w != 0) {
    return fail(MM_ERR_SHAPE, "K (" + std::to_string(k) + ") must be divisable by the memory width in K (" +
                                  std::to_string(w) + ").");
  }
  if (m % w != 0) {
    return fail(MM_ERR_SHAPE, "M (" + std::to_string(m) + ") must be divisable by the memory width in M (" +
                                  std::to_string(w) + ").");
  }
  return MM_OK;
}

// The kernels use 128-bit global accesses and TMA descriptors on A, B and C.
int check_device_alignment(const void *a, const void *b, const void *c) {
  if ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c)) % 16 != 0) {
    return fail(MM_ERR_INVALID, "device matrix pointers must be 16-byte aligned");
  }
  return MM_OK;
}

mm::GemmArgs make_args(mm_context *ctx, const void *a, const void *b, void *c, unsigned n, unsigned k, unsigned m,
                       int flags, cudaStream_t stream) {
  mm::GemmArgs g{a, b, c, n, k, m, flags, stream};
  g.tuning = &ctx->tuning;
  return g;
}

// The problems of a batched call (mm_kernel_enqueue_batched); the single-problem entries pass batch = 1,
// for which the MM_FLAG_BATCH_SHARED_* flags change nothing.
mm::GemmBatch make_batch(unsigned batch, int flags) {
  mm::GemmBatch bt;
  bt.count = batch;
  bt.shared_a = (flags & MM_FLAG_BATCH_SHARED_A) != 0;
  bt.shared_b = (flags & MM_FLAG_BATCH_SHARED_B) != 0;
  return bt;
}

// Rules of a batched call on top of check_args: batch in [1, 65535] (the kernels index problems by
// gridDim.z, at most 65535), and the stacked extents batch * N, K, M below 2^31 (TMA coordinates are
// signed 32-bit).
int check_batch(unsigned batch, unsigned n, unsigned k, unsigned m) {
  if (batch == 0) return fail(MM_ERR_INVALID, "batch must be positive");
  if (batch > 65535) {
    return fail(MM_ERR_UNSUPPORTED, "batch (" + std::to_string(batch) + ") must not exceed 65535");
  }
  const uint64_t limit = uint64_t(1) << 31;
  if (uint64_t(batch) * n >= limit || uint64_t(batch) * k >= limit || uint64_t(batch) * m >= limit) {
    return fail(MM_ERR_UNSUPPORTED, "batch * N, batch * K and batch * M must be below 2^31");
  }
  return MM_OK;
}

// Bit matrices: K and M (the closure's N) multiples of 128, so that every row is a whole number of 16-byte words.
int check_bool_shape(const char *what, unsigned x) {
  if (x % 128 != 0) {
    return fail(MM_ERR_SHAPE, std::string(what) + " (" + std::to_string(x) + ") must be a multiple of 128 bits.");
  }
  return MM_OK;
}

// Whether the byte ranges [x, x + x_bytes) and [y, y + y_bytes) share a byte.
bool overlaps(const void *x, size_t x_bytes, const void *y, size_t y_bytes) {
  const uintptr_t x0 = reinterpret_cast<uintptr_t>(x), y0 = reinterpret_cast<uintptr_t>(y);
  return x0 < y0 + y_bytes && y0 < x0 + x_bytes;
}

// Stream-capture and profiling bookkeeping of one enqueued call.  *pe = the call's three profiling events (start,
// after preparation, after the main kernel; the start one already recorded), or null when `profile` is false or
// profiling is off or full.
int begin_call(mm_context *ctx, cudaStream_t stream, bool profile, cudaStreamCaptureStatus *capture,
               cudaEvent_t **pe) {
  *capture = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(stream, capture) == cudaSuccess && *capture != cudaStreamCaptureStatusNone) {
    ctx->captured = true;
  }
  *pe = nullptr;
  if (profile && ctx->profiling && ctx->prof_calls < 256) {
    while (ctx->prof_events.size() < size_t(3 * (ctx->prof_calls + 1))) {
      cudaEvent_t e;
      MM_CUDA_TRY(cudaEventCreate(&e));
      ctx->prof_events.push_back(e);
    }
    *pe = &ctx->prof_events[3 * ctx->prof_calls];
    ++ctx->prof_calls;
    MM_CUDA_TRY(cudaEventRecord((*pe)[0], stream));
  }
  return MM_OK;
}

int enqueue_locked(mm_context *ctx, int dtype, int map_op, int reduce_op, int flags, const void *a,
                   const void *b, void *c, unsigned n, unsigned k, unsigned m, cudaStream_t stream,
                   bool dry_run = false, unsigned batch = 1, bool accumulate = false,
                   const mm::AgreeFn *agree = nullptr) {
  mm::GemmArgs g = make_args(ctx, a, b, c, n, k, m, flags, stream);
  g.agree = agree;
  g.batch = make_batch(batch, flags);
  g.dry_run = dry_run;
  g.accumulate = accumulate;
  cudaStreamCaptureStatus capture;
  cudaEvent_t *pe;
  const int rc_begin = begin_call(ctx, stream, !dry_run, &capture, &pe);
  if (rc_begin != MM_OK) return rc_begin;
  if (pe) g.ev_prep_done = pe[1];
  int rc_launch = MM_OK;
  switch (select_path(dtype, map_op, reduce_op, flags, n, k)) {
    case kPathTcgen05: {
      const size_t need = mm::tcgen05_scratch_bytes(dtype, n, k, m, flags, ctx->tuning, g.batch);
      if (need > ctx->scratch.bytes && capture != cudaStreamCaptureStatusNone) {
        return fail(MM_ERR_INVALID, batch > 1 ? "the scratch cannot grow during stream capture: call mm_context_reserve_batched() first"
                                              : "the scratch cannot grow during stream capture: call mm_context_reserve() first");
      }
      int rc = ensure(ctx, ctx->scratch, need, ctx->captured);
      if (rc != MM_OK) return rc;
      rc_launch = mm::launch_tcgen05(dtype, g, ctx->scratch.ptr, ctx->scratch.bytes);
      break;
    }
    case kPathDmma:
      if (pe) MM_CUDA_TRY(cudaEventRecord(pe[1], stream));
      rc_launch = accumulate ? mm::launch_dmma_accumulate(g) : mm::launch_dmma(g);
      break;
    case kPathSemiring:
      if (pe) MM_CUDA_TRY(cudaEventRecord(pe[1], stream));
      rc_launch = accumulate ? mm::launch_semiring_accumulate(dtype, map_op, reduce_op, g)
                             : mm::launch_semiring(dtype, map_op, reduce_op, g);
      break;
  }
  if (rc_launch != MM_OK) return rc_launch;
  if (pe) MM_CUDA_TRY(cudaEventRecord(pe[2], stream));
  return MM_OK;
}

void destroy_context(mm_context *ctx) {
  cudaSetDevice(ctx->device);
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  if (ctx->scratch.ptr) cudaFree(ctx->scratch.ptr);
  for (auto &s : ctx->staging) {
    if (s.ptr) cudaFree(s.ptr);
  }
  for (void *p : ctx->retired) cudaFree(p);
  for (auto e : ctx->prof_events) cudaEventDestroy(e);
  for (auto e : ctx->sync_events) cudaEventDestroy(e);
  for (cudaEvent_t e : {ctx->ev_start, ctx->ev_stop, ctx->ev_slice}) {
    if (e) cudaEventDestroy(e);
  }
  for (cudaStream_t s : {ctx->copy_in, ctx->copy_out, ctx->stream}) {
    if (s) cudaStreamDestroy(s);
  }
  delete ctx;
}

int init_context(mm_context *ctx) {
  MM_CUDA_TRY(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
  MM_CUDA_TRY(cudaStreamCreateWithFlags(&ctx->copy_in, cudaStreamNonBlocking));
  MM_CUDA_TRY(cudaStreamCreateWithFlags(&ctx->copy_out, cudaStreamNonBlocking));
  MM_CUDA_TRY(cudaEventCreate(&ctx->ev_start));
  MM_CUDA_TRY(cudaEventCreate(&ctx->ev_stop));
  MM_CUDA_TRY(cudaEventCreateWithFlags(&ctx->ev_slice, cudaEventDisableTiming));
  return MM_OK;
}

// ---- the pipelined host-pointer path --------------------------------------------------------------
// How B reaches the device of one pipeline.  Single GPU: the whole of B over PCIe.  Multi-GPU: this
// device uploads rows [k0, k1) only; the other slices are read from the peers' B buffers over NVLink
// (`parts_dev`: device array of the devices' B base pointers, slice j = rows [j * part_rows, ...)).
struct BPlan {
  unsigned k0 = 0, k1 = 0;
  const void *const *parts_dev = nullptr;
  unsigned part_rows = 0;
  std::vector<cudaEvent_t> peer_slices;  // the peers' "slice uploaded" events (recorded before this is used)
};

struct Pipeline {
  mm_context *ctx;
  int dtype, map_op, reduce_op, flags;
  const unsigned char *a_host;  // this pipeline's rows of A (row-major) or all of A (transposed)
  const unsigned char *b_host;  // all of B
  unsigned char *c_host;        // this pipeline's rows of C
  unsigned rows, k, m;
  size_t es;
  Path path;
  unsigned char *da = nullptr, *db = nullptr, *dc = nullptr;

  // Phase 1: allocations + this device's (slice of) B on its way.  Records ctx->ev_slice.
  int upload_b(const BPlan &bp) {
    MM_CUDA_TRY(cudaSetDevice(ctx->device));
    ++ctx->staging_gen;
    int rc;
    if ((rc = ensure(ctx, ctx->staging[0], size_t(rows) * k * es, false)) != MM_OK) return rc;
    if ((rc = ensure(ctx, ctx->staging[1], size_t(k) * m * es, false)) != MM_OK) return rc;
    if ((rc = ensure(ctx, ctx->staging[2], size_t(rows) * m * es, false)) != MM_OK) return rc;
    if (path == kPathTcgen05) {
      rc = ensure(ctx, ctx->scratch, mm::tcgen05_scratch_bytes(dtype, rows, k, m, flags, ctx->tuning), ctx->captured);
      if (rc != MM_OK) return rc;
    }
    da = static_cast<unsigned char *>(ctx->staging[0].ptr);
    db = static_cast<unsigned char *>(ctx->staging[1].ptr);
    dc = static_cast<unsigned char *>(ctx->staging[2].ptr);
    const size_t off = size_t(bp.k0) * m * es, bytes = size_t(bp.k1 - bp.k0) * m * es;
    if (bytes) MM_CUDA_TRY(cudaMemcpyAsync(db + off, b_host + off, bytes, cudaMemcpyHostToDevice, ctx->copy_in));
    MM_CUDA_TRY(cudaEventRecord(ctx->ev_slice, ctx->copy_in));
    return MM_OK;
  }

  // Phase 2: A row-chunks in, kernels, C row-chunks out; blocking.  C row-blocks are independent
  // (kernel/Compute.cpp:53-56), so the H2D copy of A chunk i+1, the kernels of chunk i and the D2H
  // copy of C chunk i-1 run concurrently on three streams; B is assembled (and, on the tcgen05 path,
  // prepared) once.  A stored K x N cannot be cut into contiguous row chunks: single chunk.
  // `agree` (multi-GPU, mm::AgreeFn): called once every A chunk of this device is prepared and before any GEMM.
  int run(const BPlan &bp, double *seconds_device, const mm::AgreeFn *agree = nullptr) {
    const int rc = enqueue_all(bp, agree);
    // drain every stream before returning, on the error paths too: the caller's host buffers must
    // not be touched by copies in flight after this call has returned
    cudaError_t e = cudaSuccess;
    for (cudaStream_t s : {ctx->copy_in, ctx->stream, ctx->copy_out}) {
      const cudaError_t es_ = cudaStreamSynchronize(s);
      if (e == cudaSuccess) e = es_;
    }
    if (rc != MM_OK) return rc;
    if (e != cudaSuccess) return fail(MM_ERR_CUDA, std::string("host pipeline: ") + cudaGetErrorString(e));
    if (seconds_device) {
      // first kernel start .. last kernel end on the compute stream (with more than one chunk this
      // includes the stalls waiting for A chunks to arrive)
      float ms = 0.f;
      MM_CUDA_TRY(cudaEventElapsedTime(&ms, ctx->ev_start, ctx->ev_stop));
      *seconds_device = 1e-3 * ms;
    }
    return MM_OK;
  }

 private:
  int enqueue_all(const BPlan &bp, const mm::AgreeFn *agree) {
    MM_CUDA_TRY(cudaSetDevice(ctx->device));
    const bool ta = (flags & MM_FLAG_TRANSPOSED_A) != 0;
    const mm::Tuning &t = ctx->tuning;
    unsigned chunk_rows = rows;
    if (!ta) {
      const size_t row_bytes = size_t(k) * es;
      size_t cr = std::max<size_t>((rows + 15) / 16, ((size_t(32) << 20) + row_bytes - 1) / row_bytes);
      if (const char *e = std::getenv("MM_HOST_CHUNK_ROWS")) cr = std::max(1, std::atoi(e));  // tests force small chunks
      cr = (cr + 127) / 128 * 128;
      if (cr < rows) chunk_rows = unsigned(cr);
    }
    const unsigned chunks = (rows + chunk_rows - 1) / chunk_rows;
    while (ctx->sync_events.size() < size_t(2 * chunks)) {
      cudaEvent_t e;
      MM_CUDA_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
      ctx->sync_events.push_back(e);
    }
    auto ev_a = [&](unsigned i) { return ctx->sync_events[i]; };
    auto ev_c = [&](unsigned i) { return ctx->sync_events[chunks + i]; };

    // ---- H2D stream: A chunks (B's slice went first, in upload_b)
    for (unsigned i = 0; i < chunks; ++i) {
      const size_t r0 = size_t(i) * chunk_rows, nr = std::min<size_t>(chunk_rows, rows - r0);
      if (!ta) {
        MM_CUDA_TRY(cudaMemcpyAsync(da + r0 * k * es, a_host + r0 * k * es, nr * k * es, cudaMemcpyHostToDevice,
                                    ctx->copy_in));
      } else {
        MM_CUDA_TRY(cudaMemcpyAsync(da, a_host, size_t(rows) * k * es, cudaMemcpyHostToDevice, ctx->copy_in));
      }
      MM_CUDA_TRY(cudaEventRecord(ev_a(i), ctx->copy_in));
    }

    // ---- compute stream: B complete on this device (own slice + the peers' slices in place)
    MM_CUDA_TRY(cudaStreamWaitEvent(ctx->stream, ctx->ev_slice, 0));
    for (cudaEvent_t e : bp.peer_slices) MM_CUDA_TRY(cudaStreamWaitEvent(ctx->stream, e, 0));
    MM_CUDA_TRY(cudaEventRecord(ctx->ev_start, ctx->stream));
    int rc = MM_OK;
    if (bp.parts_dev != nullptr) {  // also with a single slice: the GPUs that did not upload it read it from its owner
      rc = mm::gather_b_rows(bp.parts_dev, bp.part_rows, db, es, k, m, ctx->stream);  // the peers' slices, over NVLink
      if (rc != MM_OK) return rc;
    }
    const void *b_op = nullptr;
    unsigned char *aprep = nullptr;
    mm::HalfScratch hs;
    if (path == kPathTcgen05) {
      hs = mm::tcgen05_half_scratch(ctx->scratch.ptr, ctx->scratch.bytes, dtype, rows, k, m, flags, t);
      if (hs.fits_b) {
        // float: the one-pass preparation of B
        MM_CUDA_TRY(cudaMemsetAsync(hs.fits_b, 1, hs.flag_bytes, ctx->stream));
        rc = mm::tcgen05_prepare_float(false, nullptr, 0, 0, db, rows, k, m, flags, t, mm::GemmBatch{},
                                       ctx->scratch.ptr, ctx->scratch.bytes, ctx->stream);
        b_op = ctx->scratch.ptr;
      } else {
        rc = mm::tcgen05_prepare_b(dtype, db, ctx->scratch.ptr, k, m, flags, t, &b_op, ctx->stream);
      }
      if (rc != MM_OK) return rc;
      aprep = static_cast<unsigned char *>(ctx->scratch.ptr) + mm::tcgen05_bt_bytes(dtype, k, m, flags, t);
    }
    // With fp16 copies every chunk's preparation clears the one fits flag of A, and the GEMMs start once all of A is
    // prepared and the TF32 copies still owed are written: each chunk then takes the datapath of the whole A, so the
    // chunks' C is the single call's, bit for bit.
    const bool prepare_first = hs.fits_a != nullptr;
    std::vector<const void *> a_ops(chunks);
    auto prepare = [&](unsigned i) -> int {
      const size_t r0 = size_t(i) * chunk_rows, nr = std::min<size_t>(chunk_rows, rows - r0);
      MM_CUDA_TRY(cudaStreamWaitEvent(ctx->stream, ev_a(i), 0));
      if (path != kPathTcgen05) return MM_OK;
      if (hs.fits_a != nullptr) {
        a_ops[i] = aprep + r0 * k * es;
        return mm::tcgen05_prepare_float(false, da + (ta ? 0 : r0 * k * es), unsigned(r0), unsigned(nr), nullptr, rows,
                                         k, m, flags, t, mm::GemmBatch{}, ctx->scratch.ptr, ctx->scratch.bytes,
                                         ctx->stream);
      }
      const size_t a_scale = (dtype == MM_DTYPE_FLOAT && (flags & MM_FLAG_TF32X3)) ? 3 : 1;
      return mm::tcgen05_prepare_a(dtype, da + (ta ? 0 : r0 * k * es), aprep + (ta ? 0 : r0 * k * es * a_scale),
                                   unsigned(nr), k, flags, t, &a_ops[i], ctx->stream, 1);
    };
    auto compute = [&](unsigned i) -> int {
      const size_t r0 = size_t(i) * chunk_rows, nr = std::min<size_t>(chunk_rows, rows - r0);
      const void *a_chunk = da + (ta ? 0 : r0 * k * es);
      void *c_chunk = dc + r0 * m * es;
      int rc1;
      if (path == kPathTcgen05) {
        mm::HalfOperands half = hs.operands();
        if (half.a) half.a = static_cast<const unsigned char *>(half.a) + r0 * k * 2;
        rc1 = mm::tcgen05_gemm(dtype, a_ops[i], b_op, c_chunk, unsigned(nr), k, m, flags, t,
                               mm::tcgen05_tile_sync(ctx->scratch.ptr, ctx->scratch.bytes), ctx->stream,
                               mm::GemmBatch{}, false, half);
      } else {
        mm::GemmArgs g = make_args(ctx, a_chunk, db, c_chunk, unsigned(nr), k, m, flags, ctx->stream);
        rc1 = (path == kPathDmma) ? mm::launch_dmma(g) : mm::launch_semiring(dtype, map_op, reduce_op, g);
      }
      if (rc1 == MM_OK) MM_CUDA_TRY(cudaEventRecord(ev_c(i), ctx->stream));
      return rc1;
    };
    if (prepare_first) {
      for (unsigned i = 0; i < chunks && rc == MM_OK; ++i) rc = prepare(i);
    }
    if (rc == MM_OK && agree != nullptr) rc = (*agree)(hs.fits_a, ctx->stream);
    if (rc == MM_OK && prepare_first) {  // one second pass over B and all of A
      rc = mm::tcgen05_prepare_float(true, da, 0, rows, db, rows, k, m, flags, t, mm::GemmBatch{}, ctx->scratch.ptr,
                                     ctx->scratch.bytes, ctx->stream);
    }
    for (unsigned i = 0; i < chunks && rc == MM_OK; ++i) {
      if (!prepare_first) rc = prepare(i);
      if (rc == MM_OK) rc = compute(i);
    }
    if (rc != MM_OK) return rc;
    MM_CUDA_TRY(cudaEventRecord(ctx->ev_stop, ctx->stream));

    // ---- D2H stream
    for (unsigned i = 0; i < chunks; ++i) {
      const size_t r0 = size_t(i) * chunk_rows, nr = std::min<size_t>(chunk_rows, rows - r0);
      MM_CUDA_TRY(cudaStreamWaitEvent(ctx->copy_out, ev_c(i), 0));
      MM_CUDA_TRY(cudaMemcpyAsync(c_host + r0 * m * es, dc + r0 * m * es, nr * m * es, cudaMemcpyDeviceToHost,
                                  ctx->copy_out));
    }
    return MM_OK;
  }
};

std::mutex g_default_mutex;
mm_context *g_default_ctx = nullptr;
mm_multi *g_default_multi = nullptr;

int env_int(const char *name, int fallback) {
  const char *e = std::getenv(name);
  return (e && *e) ? std::atoi(e) : fallback;
}

// Reusable host barrier for the worker threads of one multi-GPU call.
class HostBarrier {
 public:
  explicit HostBarrier(int n) : n_(n) {}
  void arrive_and_wait() {
    std::unique_lock<std::mutex> lock(m_);
    const int gen = gen_;
    if (++count_ == n_) {
      count_ = 0;
      ++gen_;
      cv_.notify_all();
    } else {
      cv_.wait(lock, [&] { return gen_ != gen; });
    }
  }

 private:
  std::mutex m_;
  std::condition_variable cv_;
  int n_, count_ = 0, gen_ = 0;
};

// The float datapath of a multi-GPU call is the one the single call on the whole A takes (DESIGN.md §3.1): each
// device reads its fits word of A once its rows are prepared, and every device clears its word unless all of them
// fit.  agree(g) is device g's mm::AgreeFn; every device must pass the barrier once, so finish(g) passes it for a
// device whose call never got as far (no rows, another kernel family, an error).
class FitsAgreement {
 public:
  FitsAgreement(HostBarrier &barrier, int gpus) : barrier_(barrier), fit_(gpus, 1), agreed_(gpus, 0) {}
  mm::AgreeFn agree(int g) {
    return [this, g](unsigned int *fits, cudaStream_t stream) -> int {
      agreed_[g] = 1;
      int rc = MM_OK;
      unsigned int v = 1;
      if (fits != nullptr) {
        cudaError_t e = cudaStreamSynchronize(stream);  // this device's A is prepared
        if (e == cudaSuccess) e = cudaMemcpy(&v, fits, sizeof(v), cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) rc = fail(MM_ERR_CUDA, std::string("reading the fits word of A: ") + cudaGetErrorString(e));
      }
      fit_[g] = v != 0u;
      barrier_.arrive_and_wait();
      const bool all = std::all_of(fit_.begin(), fit_.end(), [](int f) { return f != 0; });
      if (rc == MM_OK && fits != nullptr && v != 0u && !all) MM_CUDA_TRY(cudaMemsetAsync(fits, 0, sizeof(v), stream));
      return rc;
    };
  }
  void finish(int g) {
    if (!agreed_[g]) barrier_.arrive_and_wait();
  }

 private:
  HostBarrier &barrier_;
  std::vector<int> fit_;      // per device: its rows of A fit (1 for a device without a fits word)
  std::vector<char> agreed_;  // per device: agree() ran
};

}  // namespace

struct mm_multi {
  std::vector<mm_context *> ctx;
  std::vector<void **> parts_dev;  // per device: device array of G pointers to the devices' B buffers
  bool peer = false;
  std::mutex mutex;
  // resident problem of the upload / execute / download lifecycle: valid while every device's staging
  // generation is the one its upload left (no other call has written those buffers since)
  unsigned n = 0, k = 0, m = 0;
  int dtype = -1;
  std::vector<uint64_t> gen;
  bool executed = false;  // an execute has run on the resident operands since the upload
};

namespace {

unsigned rows_per_gpu(unsigned n, int g) { return (n + unsigned(g) - 1) / unsigned(g); }

// The partition rule of every mm_multi_* entry (and of mm_multi_partition): rows of A / C, K-row slices of B.
struct Partition {
  unsigned r0, r1;   // rows of A and C owned by the GPU
  unsigned k0, k1;   // K-rows of B it uploads
  unsigned part_rows, parts;
};
Partition partition_for(int gpus, int g, unsigned n, unsigned k, bool sliced_b) {
  Partition p;
  const unsigned per = rows_per_gpu(n, gpus);
  p.r0 = std::min(n, unsigned(g) * per);
  p.r1 = std::min(n, p.r0 + per);
  // B row-slices: multiples of 64 k-rows so that a preparation work item never straddles two GPUs
  p.part_rows = sliced_b ? std::max(64u, (rows_per_gpu(k, gpus) + 63u) / 64u * 64u) : k;
  p.parts = sliced_b ? (k + p.part_rows - 1) / p.part_rows : 1;
  if (sliced_b) {
    p.k0 = std::min(k, unsigned(g) * p.part_rows);
    p.k1 = (unsigned(g) >= p.parts) ? p.k0 : std::min(k, p.k0 + p.part_rows);   // more GPUs than slices: nothing to upload
  } else {
    p.k0 = 0;
    p.k1 = k;
  }
  return p;
}

// Runs fn(g) on one host thread per device; returns the first error (message re-set on this thread).
template <class Fn>
int fan_out(int gpus, Fn fn) {
  std::vector<int> rc(gpus, MM_OK);
  std::vector<std::string> msg(gpus);
  std::vector<std::thread> pool;
  for (int g = 0; g < gpus; ++g) {
    pool.emplace_back([&, g] {
      rc[g] = fn(g);
      if (rc[g] != MM_OK) msg[g] = mm_last_error();
    });
  }
  for (auto &t : pool) t.join();
  for (int g = 0; g < gpus; ++g) {
    if (rc[g] != MM_OK) return fail(rc[g], "GPU " + std::to_string(g) + ": " + msg[g]);
  }
  return MM_OK;
}

// Point every device's slice table at the devices' current B buffers (they move when they grow).
int refresh_parts(mm_multi *mu, int g) {
  mm_context *ctx = mu->ctx[g];
  MM_CUDA_TRY(cudaSetDevice(ctx->device));
  std::vector<void *> table(mu->ctx.size());
  for (size_t j = 0; j < mu->ctx.size(); ++j) table[j] = mu->ctx[j]->staging[1].ptr;
  MM_CUDA_TRY(cudaMemcpy(mu->parts_dev[g], table.data(), table.size() * sizeof(void *), cudaMemcpyHostToDevice));
  return MM_OK;
}

int multi_gemm_host_locked(mm_multi *mu, int dtype, int map_op, int reduce_op, int flags, const void *a, const void *b,
                           void *c, unsigned n, unsigned k, unsigned m, double *seconds_device) {
  if (flags & MM_FLAG_TRANSPOSED_A) {
    return fail(MM_ERR_UNSUPPORTED, "the row-block split over GPUs needs row-major A (MM_TRANSPOSED_A is set)");
  }
  const int G = int(mu->ctx.size());
  const size_t es = mm_dtype_size(dtype);
  std::vector<Pipeline> pipes(G);
  std::vector<BPlan> plans(G);
  std::vector<double> dev_s(G, 0.0);
  HostBarrier barrier(G);
  FitsAgreement fits(barrier, G);
  int rc = fan_out(G, [&](int g) -> int {
    const Partition part = partition_for(G, g, n, k, mu->peer);
    const unsigned r0 = part.r0, r1 = part.r1;
    Pipeline &p = pipes[g];
    p = Pipeline{mu->ctx[g], dtype, map_op, reduce_op, flags,
                 static_cast<const unsigned char *>(a) + size_t(r0) * k * es, static_cast<const unsigned char *>(b),
                 static_cast<unsigned char *>(c) + size_t(r0) * m * es, r1 - r0, k, m, es,
                 select_path(dtype, map_op, reduce_op, flags, std::max(1u, r1 - r0), k)};
    BPlan &bp = plans[g];
    bp.k0 = part.k0;
    bp.k1 = part.k1;
    if (mu->peer) {
      bp.part_rows = part.part_rows;
      bp.parts_dev = mu->parts_dev[g];
    }
    std::lock_guard<std::mutex> lock(mu->ctx[g]->mutex);
    // a GPU without rows still uploads its slice of B: the others read it
    if (p.rows == 0) p.rows = 1, p.a_host = static_cast<const unsigned char *>(a), p.c_host = nullptr;
    int rc1 = p.upload_b(bp);
    barrier.arrive_and_wait();  // every slice event is recorded and every B buffer has its final address
    int rc2 = (rc1 == MM_OK && mu->peer) ? refresh_parts(mu, g) : MM_OK;
    if (mu->peer) {
      for (int j = 0; j < G; ++j) {
        if (j != g) bp.peer_slices.push_back(mu->ctx[j]->ev_slice);
      }
    }
    barrier.arrive_and_wait();  // all slice tables are in place before any kernel dereferences one
    const mm::AgreeFn agree = fits.agree(g);
    int rc3 = MM_OK;
    if (rc1 == MM_OK && rc2 == MM_OK && r1 > r0) {
      rc3 = p.run(bp, &dev_s[g], &agree);
    } else {
      cudaSetDevice(mu->ctx[g]->device);
      cudaStreamSynchronize(mu->ctx[g]->copy_in);
    }
    fits.finish(g);
    // nobody's B buffer may be reused (next call) before every peer has finished reading it
    barrier.arrive_and_wait();
    return rc1 != MM_OK ? rc1 : (rc2 != MM_OK ? rc2 : rc3);
  });
  if (rc != MM_OK) return rc;
  if (seconds_device) *seconds_device = *std::max_element(dev_s.begin(), dev_s.end());
  return MM_OK;
}

void clear_resident(mm_multi *mu) {
  mu->n = mu->k = mu->m = 0;
  mu->dtype = -1;
  mu->gen.clear();
  mu->executed = false;
}

// The resident problem of mm_multi_upload is (dtype, n, k, m) and still sits in every device's staging buffers.
int check_resident(mm_multi *mu, const char *entry, int dtype, unsigned n, unsigned k, unsigned m) {
  if (mu->dtype != dtype || mu->n != n || mu->k != k || mu->m != m) {
    return fail(MM_ERR_INVALID, std::string(entry) + ": no matching mm_multi_upload (type or sizes differ)");
  }
  for (size_t g = 0; g < mu->ctx.size(); ++g) {
    std::lock_guard<std::mutex> lock(mu->ctx[g]->mutex);
    if (mu->ctx[g]->staging_gen != mu->gen[g]) {
      return fail(MM_ERR_INVALID, std::string(entry) + ": no matching mm_multi_upload (GPU " + std::to_string(g) +
                                      "'s buffers were reused by another call since)");
    }
  }
  return MM_OK;
}

int create_multi(int n_gpus, const int *devices, mm_multi **out) {
  mm_multi *mu = new mm_multi();
  auto cleanup = [&](int rc) {
    const std::string msg = mm_last_error();
    mm_multi_destroy(mu);
    mm::set_error(msg);
    return rc;
  };
  for (int g = 0; g < n_gpus; ++g) {
    mm_context *c = nullptr;
    const int rc = mm_context_create(devices ? devices[g] : g, &c);
    if (rc != MM_OK) return cleanup(rc);
    mu->ctx.push_back(c);
  }
  mu->peer = n_gpus > 1;
  for (int g = 0; g < n_gpus && mu->peer; ++g) {
    for (int j = 0; j < n_gpus; ++j) {
      if (mu->ctx[j]->device == mu->ctx[g]->device) continue;  // the same device twice (tests): plain local memory
      int can = 0;
      if (cudaDeviceCanAccessPeer(&can, mu->ctx[g]->device, mu->ctx[j]->device) != cudaSuccess || !can) mu->peer = false;
    }
  }
  for (int g = 0; g < n_gpus; ++g) {
    if (cudaSetDevice(mu->ctx[g]->device) != cudaSuccess) return cleanup(fail(MM_ERR_CUDA, "cudaSetDevice failed"));
    for (int j = 0; j < n_gpus && mu->peer; ++j) {
      if (mu->ctx[j]->device == mu->ctx[g]->device) continue;
      const cudaError_t e = cudaDeviceEnablePeerAccess(mu->ctx[j]->device, 0);
      if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
      else if (e != cudaSuccess) mu->peer = false;
    }
    void **table = nullptr;
    if (cudaMalloc(&table, sizeof(void *) * size_t(n_gpus)) != cudaSuccess) {
      return cleanup(fail(MM_ERR_NOMEM, "cudaMalloc of the slice table failed"));
    }
    mu->parts_dev.push_back(table);
  }
  *out = mu;
  return MM_OK;
}

// mm_kernel_execute; `agree` as in GemmArgs (mm_multi_execute), passed to the real launch only.
int kernel_execute(mm_context *ctx, int dtype, int map_op, int reduce_op, int flags, const void *a, const void *b,
                   void *c, unsigned n, unsigned k, unsigned m, double *seconds_device, double *seconds_wall,
                   const mm::AgreeFn *agree) {
  if (!ctx) return fail(MM_ERR_INVALID, "null context");
  int rc = check_args(dtype, map_op, reduce_op, a, b, c, n, k, m);
  if (rc != MM_OK) return rc;
  if ((rc = check_device_alignment(a, b, c)) != MM_OK) return rc;
  std::lock_guard<std::mutex> lock(ctx->mutex);
  MM_CUDA_TRY(cudaSetDevice(ctx->device));
  // allocate scratch / load kernels first: the device time below is kernel time only, like the
  // OpenCL profiling interval of the reference's ExecuteTask (common/OpenCL.h:1495-1500)
  rc = enqueue_locked(ctx, dtype, map_op, reduce_op, flags, a, b, c, n, k, m, ctx->stream, /*dry_run=*/true);
  if (rc != MM_OK) return rc;
  const auto t0 = std::chrono::high_resolution_clock::now();
  MM_CUDA_TRY(cudaEventRecord(ctx->ev_start, ctx->stream));
  rc = enqueue_locked(ctx, dtype, map_op, reduce_op, flags, a, b, c, n, k, m, ctx->stream, false, 1, false, agree);
  if (rc != MM_OK) {
    cudaStreamSynchronize(ctx->stream);
    return rc;
  }
  MM_CUDA_TRY(cudaEventRecord(ctx->ev_stop, ctx->stream));
  MM_CUDA_TRY(cudaEventSynchronize(ctx->ev_stop));
  const auto t1 = std::chrono::high_resolution_clock::now();
  float ms = 0.f;
  MM_CUDA_TRY(cudaEventElapsedTime(&ms, ctx->ev_start, ctx->ev_stop));
  if (seconds_device) *seconds_device = 1e-3 * ms;
  if (seconds_wall) *seconds_wall = std::chrono::duration<double>(t1 - t0).count();
  return MM_OK;
}

}  // namespace

extern "C" {

const char *mm_last_error(void) { return mm::g_last_error.c_str(); }

int mm_version(void) { return 203; }

size_t mm_dtype_size(int dtype) {
  switch (dtype) {
    case MM_DTYPE_HALF: return 2;
    case MM_DTYPE_FLOAT: return 4;
    case MM_DTYPE_DOUBLE: return 8;
    case MM_DTYPE_INT32: return 4;
    case MM_DTYPE_UINT32: return 4;
    case MM_DTYPE_UINT8: return 1;
    case MM_DTYPE_BFLOAT16: return 2;
  }
  return 0;
}

unsigned mm_memory_width(int dtype) {
  const size_t s = mm_dtype_size(dtype);
  return s ? static_cast<unsigned>(64 / s) : 0;
}

int mm_context_create(int device, mm_context **out) {
  if (!out) return fail(MM_ERR_INVALID, "null output pointer");
  *out = nullptr;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) {
    return fail(MM_ERR_CUDA, std::string("no CUDA device available: ") +
                                 (e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0"));
  }
  if (device < 0 || device >= count) return fail(MM_ERR_INVALID, "device ordinal out of range");
  MM_CUDA_TRY(cudaSetDevice(device));
  cudaDeviceProp prop;
  MM_CUDA_TRY(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    return fail(MM_ERR_UNSUPPORTED, std::string("libmm_b200 is built for sm_90a only; device is sm_") +
                                        std::to_string(prop.major) + std::to_string(prop.minor));
  }
  mm_context *ctx = new mm_context();
  ctx->device = device;
  ctx->tuning = mm::default_tuning();
  const int rc = init_context(ctx);
  if (rc != MM_OK) {
    const std::string msg = mm_last_error();
    destroy_context(ctx);  // releases whatever was created before the failure
    mm::set_error(msg);
    return rc;
  }
  *out = ctx;
  return MM_OK;
}

int mm_context_destroy(mm_context *ctx) {
  if (!ctx) return MM_OK;
  destroy_context(ctx);
  return MM_OK;
}

int mm_context_set_tuning(mm_context *ctx, int knob, int value) {
  if (!ctx) return fail(MM_ERR_INVALID, "null context");
  const int rc = mm::tuning_validate(knob, value);
  if (rc != MM_OK) return rc;
  std::lock_guard<std::mutex> lock(ctx->mutex);
  ctx->tuning.v[knob] = value;
  return MM_OK;
}

int mm_context_get_tuning(mm_context *ctx, int knob, int *value) {
  if (!ctx || !value) return fail(MM_ERR_INVALID, "null argument");
  if (knob < 0 || knob >= MM_TUNE_COUNT) return fail(MM_ERR_INVALID, "unknown tuning knob " + std::to_string(knob));
  std::lock_guard<std::mutex> lock(ctx->mutex);
  *value = ctx->tuning.v[knob];
  return MM_OK;
}

int mm_context_reserve(mm_context *ctx, int dtype, int flags, unsigned n, unsigned k, unsigned m) {
  if (!ctx) return fail(MM_ERR_INVALID, "null context");
  if (!valid_dtype(dtype)) return fail(MM_ERR_INVALID, "unknown MM_DATA_TYPE code");
  std::lock_guard<std::mutex> lock(ctx->mutex);
  MM_CUDA_TRY(cudaSetDevice(ctx->device));
  if (!tensor_core_dtype(dtype)) return MM_OK;  // only the tcgen05 path keeps scratch
  return ensure(ctx, ctx->scratch, mm::tcgen05_scratch_bytes(dtype, n, k, m, flags & ~MM_FLAG_EXACT, ctx->tuning),
                ctx->captured);
}

int mm_context_reserve_batched(mm_context *ctx, int dtype, int flags, unsigned n, unsigned k, unsigned m,
                               unsigned batch) {
  if (!ctx) return fail(MM_ERR_INVALID, "null context");
  if (!valid_dtype(dtype)) return fail(MM_ERR_INVALID, "unknown MM_DATA_TYPE code");
  int rc = check_batch(batch, n, k, m);
  if (rc != MM_OK) return rc;
  std::lock_guard<std::mutex> lock(ctx->mutex);
  MM_CUDA_TRY(cudaSetDevice(ctx->device));
  if (!tensor_core_dtype(dtype)) return MM_OK;  // only the tcgen05 path keeps scratch
  const int f = flags & ~MM_FLAG_EXACT;
  return ensure(ctx, ctx->scratch, mm::tcgen05_scratch_bytes(dtype, n, k, m, f, ctx->tuning, make_batch(batch, f)),
                ctx->captured);
}

int mm_buffer_alloc(mm_context *ctx, size_t bytes, void **device_ptr) {
  if (!ctx || !device_ptr) return fail(MM_ERR_INVALID, "null argument");
  *device_ptr = nullptr;
  MM_CUDA_TRY(cudaSetDevice(ctx->device));
  cudaError_t e = cudaMalloc(device_ptr, bytes ? bytes : 1);
  if (e != cudaSuccess) {
    return fail(e == cudaErrorMemoryAllocation ? MM_ERR_NOMEM : MM_ERR_CUDA,
                std::string("cudaMalloc: ") + cudaGetErrorString(e));
  }
  return MM_OK;
}

int mm_buffer_free(mm_context *ctx, void *device_ptr) {
  if (!ctx) return fail(MM_ERR_INVALID, "null context");
  MM_CUDA_TRY(cudaSetDevice(ctx->device));
  MM_CUDA_TRY(cudaFree(device_ptr));
  return MM_OK;
}

int mm_copy_to_device(mm_context *ctx, void *device_dst, const void *host_src, size_t bytes) {
  if (!ctx || !device_dst || !host_src) return fail(MM_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lock(ctx->mutex);
  MM_CUDA_TRY(cudaSetDevice(ctx->device));
  MM_CUDA_TRY(cudaMemcpyAsync(device_dst, host_src, bytes, cudaMemcpyHostToDevice, ctx->stream));
  MM_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  return MM_OK;
}

int mm_copy_to_host(mm_context *ctx, void *host_dst, const void *device_src, size_t bytes) {
  if (!ctx || !host_dst || !device_src) return fail(MM_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lock(ctx->mutex);
  MM_CUDA_TRY(cudaSetDevice(ctx->device));
  MM_CUDA_TRY(cudaMemcpyAsync(host_dst, device_src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  MM_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  return MM_OK;
}

int mm_kernel_enqueue(mm_context *ctx, int dtype, int map_op, int reduce_op, int flags,
                      const void *a, const void *b, void *c, unsigned n, unsigned k, unsigned m,
                      void *cuda_stream) {
  if (!ctx) return fail(MM_ERR_INVALID, "null context");
  int rc = check_args(dtype, map_op, reduce_op, a, b, c, n, k, m);
  if (rc != MM_OK) return rc;
  if ((rc = check_device_alignment(a, b, c)) != MM_OK) return rc;
  std::lock_guard<std::mutex> lock(ctx->mutex);
  MM_CUDA_TRY(cudaSetDevice(ctx->device));
  cudaStream_t s = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : ctx->stream;
  return enqueue_locked(ctx, dtype, map_op, reduce_op, flags, a, b, c, n, k, m, s);
}

int mm_kernel_enqueue_batched(mm_context *ctx, int dtype, int map_op, int reduce_op, int flags, const void *a,
                              const void *b, void *c, unsigned n, unsigned k, unsigned m, unsigned batch,
                              void *cuda_stream) {
  if (!ctx) return fail(MM_ERR_INVALID, "null context");
  int rc = check_args(dtype, map_op, reduce_op, a, b, c, n, k, m);
  if (rc != MM_OK) return rc;
  if ((rc = check_batch(batch, n, k, m)) != MM_OK) return rc;
  // every problem of a packed batch starts 16-byte aligned: K * sizeof(T) and M * sizeof(T) are multiples of 64
  if ((rc = check_device_alignment(a, b, c)) != MM_OK) return rc;
  std::lock_guard<std::mutex> lock(ctx->mutex);
  MM_CUDA_TRY(cudaSetDevice(ctx->device));
  cudaStream_t s = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : ctx->stream;
  return enqueue_locked(ctx, dtype, map_op, reduce_op, flags, a, b, c, n, k, m, s, /*dry_run=*/false, batch);
}

int mm_kernel_enqueue_accumulate(mm_context *ctx, int dtype, int map_op, int reduce_op, int flags, const void *a,
                                 const void *b, void *c, unsigned n, unsigned k, unsigned m, unsigned batch,
                                 void *cuda_stream) {
  if (!ctx) return fail(MM_ERR_INVALID, "null context");
  int rc = check_args(dtype, map_op, reduce_op, a, b, c, n, k, m);
  if (rc != MM_OK) return rc;
  if ((rc = check_batch(batch, n, k, m)) != MM_OK) return rc;
  if ((rc = check_device_alignment(a, b, c)) != MM_OK) return rc;
  // C is read and written while A and B are read: an overlap would feed updated elements back into the product
  const size_t es = mm_dtype_size(dtype);
  const mm::GemmBatch bt = make_batch(batch, flags);
  if (overlaps(c, size_t(batch) * n * m * es, a, size_t(bt.a_copies()) * n * k * es) ||
      overlaps(c, size_t(batch) * n * m * es, b, size_t(bt.b_copies()) * k * m * es)) {
    return fail(MM_ERR_INVALID, "C must not overlap A or B in an accumulating call");
  }
  std::lock_guard<std::mutex> lock(ctx->mutex);
  MM_CUDA_TRY(cudaSetDevice(ctx->device));
  cudaStream_t s = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : ctx->stream;
  return enqueue_locked(ctx, dtype, map_op, reduce_op, flags, a, b, c, n, k, m, s, /*dry_run=*/false, batch,
                        /*accumulate=*/true);
}

int mm_kernel_enqueue_witness(mm_context *ctx, int dtype, int map_op, int reduce_op, int flags, const void *a,
                              const void *b, void *c, unsigned *w, unsigned n, unsigned k, unsigned m, unsigned batch,
                              void *cuda_stream) {
  if (!ctx) return fail(MM_ERR_INVALID, "null context");
  int rc = check_args(dtype, map_op, reduce_op, a, b, c, n, k, m);
  if (rc != MM_OK) return rc;
  if ((rc = check_batch(batch, n, k, m)) != MM_OK) return rc;
  if ((rc = check_device_alignment(a, b, c)) != MM_OK) return rc;
  if (!w) return fail(MM_ERR_INVALID, "null witness pointer");
  if (reinterpret_cast<uintptr_t>(w) % 16 != 0) return fail(MM_ERR_INVALID, "the witness pointer must be 16-byte aligned");
  if (reduce_op != MM_OP_MIN && reduce_op != MM_OP_MAX) {
    return fail(MM_ERR_INVALID, "witnesses exist for the Min and Max reduces only");
  }
  std::lock_guard<std::mutex> lock(ctx->mutex);
  MM_CUDA_TRY(cudaSetDevice(ctx->device));
  cudaStream_t s = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : ctx->stream;
  mm::GemmArgs g = make_args(ctx, a, b, c, n, k, m, flags, s);
  g.batch = make_batch(batch, flags);
  cudaStreamCaptureStatus capture;
  cudaEvent_t *pe;
  if ((rc = begin_call(ctx, s, /*profile=*/true, &capture, &pe)) != MM_OK) return rc;
  if (pe) MM_CUDA_TRY(cudaEventRecord(pe[1], s));  // like a semiring call: no preparation
  if ((rc = mm::launch_semiring_witness(dtype, map_op, reduce_op, g, w)) != MM_OK) return rc;
  if (pe) MM_CUDA_TRY(cudaEventRecord(pe[2], s));
  return MM_OK;
}

unsigned mm_closure_block(int dtype) { return valid_dtype(dtype) ? 128u : 0u; }

int mm_kernel_enqueue_closure(mm_context *ctx, int dtype, int map_op, int reduce_op, int flags, void *d, unsigned n,
                              unsigned batch, void *cuda_stream) {
  if (!ctx) return fail(MM_ERR_INVALID, "null context");
  // D is A, B and C of an N x N x N problem: the witness call's checks with K = M = N
  int rc = check_args(dtype, map_op, reduce_op, d, d, d, n, n, n);
  if (rc != MM_OK) return rc;
  if ((rc = check_batch(batch, n, n, n)) != MM_OK) return rc;
  if ((rc = check_device_alignment(d, d, d)) != MM_OK) return rc;
  if (reduce_op != MM_OP_MIN && reduce_op != MM_OP_MAX) {
    return fail(MM_ERR_INVALID, "closures exist for the Min and Max reduces only");
  }
  if (flags & (MM_FLAG_TRANSPOSED_A | MM_FLAG_BATCH_SHARED_A | MM_FLAG_BATCH_SHARED_B)) {
    return fail(MM_ERR_INVALID, "a closure takes neither MM_FLAG_TRANSPOSED_A nor MM_FLAG_BATCH_SHARED_A / _B");
  }
  std::lock_guard<std::mutex> lock(ctx->mutex);
  MM_CUDA_TRY(cudaSetDevice(ctx->device));
  cudaStream_t s = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : ctx->stream;
  cudaStreamCaptureStatus capture;
  cudaEvent_t *pe;
  if ((rc = begin_call(ctx, s, /*profile=*/true, &capture, &pe)) != MM_OK) return rc;
  if (pe) MM_CUDA_TRY(cudaEventRecord(pe[1], s));  // like a semiring call: no preparation
  if ((rc = mm::launch_semiring_closure(dtype, map_op, reduce_op, flags, d, n, batch, s)) != MM_OK) return rc;
  if (pe) MM_CUDA_TRY(cudaEventRecord(pe[2], s));
  return MM_OK;
}

int mm_kernel_enqueue_bool(mm_context *ctx, int flags, const void *a, const void *b, void *c, unsigned n, unsigned k,
                           unsigned m, unsigned batch, void *cuda_stream) {
  if (!ctx) return fail(MM_ERR_INVALID, "null context");
  if (!a || !b || !c) return fail(MM_ERR_INVALID, "null matrix pointer");
  if (n == 0 || k == 0 || m == 0) return fail(MM_ERR_INVALID, "matrix dimensions must be positive");
  int rc;
  if ((rc = check_bool_shape("K", k)) != MM_OK || (rc = check_bool_shape("M", m)) != MM_OK) return rc;
  if ((rc = check_batch(batch, n, k, m)) != MM_OK) return rc;
  if ((rc = check_device_alignment(a, b, c)) != MM_OK) return rc;
  if (flags != 0) return fail(MM_ERR_INVALID, "flags is reserved and must be 0");
  const size_t a_bytes = size_t(batch) * n * (k / 8), b_bytes = size_t(batch) * k * (m / 8);
  const size_t c_bytes = size_t(batch) * n * (m / 8);
  if (overlaps(c, c_bytes, a, a_bytes) || overlaps(c, c_bytes, b, b_bytes)) {
    return fail(MM_ERR_INVALID, "C must not overlap A or B");
  }
  std::lock_guard<std::mutex> lock(ctx->mutex);
  MM_CUDA_TRY(cudaSetDevice(ctx->device));
  cudaStream_t s = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : ctx->stream;
  cudaStreamCaptureStatus capture;
  cudaEvent_t *pe;
  if ((rc = begin_call(ctx, s, /*profile=*/true, &capture, &pe)) != MM_OK) return rc;
  // the scratch: B's K-major copy (b_bytes), then the GEMM's wave-barrier counter at the tail
  const size_t need = b_bytes + mm::kTcgen05TailBytes;
  if (need > ctx->scratch.bytes && capture != cudaStreamCaptureStatusNone) {
    return fail(MM_ERR_INVALID, "the scratch cannot grow during stream capture: make a first call outside the capture");
  }
  if ((rc = ensure(ctx, ctx->scratch, need, ctx->captured)) != MM_OK) return rc;
  if ((rc = mm::bool_transpose_b(b, ctx->scratch.ptr, k, m, batch, s)) != MM_OK) return rc;
  if (pe) MM_CUDA_TRY(cudaEventRecord(pe[1], s));
  rc = mm::bool_gemm(a, ctx->scratch.ptr, c, n, k, m, batch, ctx->tuning,
                     mm::tcgen05_tile_sync(ctx->scratch.ptr, ctx->scratch.bytes), s);
  if (rc != MM_OK) return rc;
  if (pe) MM_CUDA_TRY(cudaEventRecord(pe[2], s));
  return MM_OK;
}

int mm_kernel_enqueue_bool_closure(mm_context *ctx, int flags, void *d, unsigned n, unsigned batch, void *cuda_stream) {
  if (!ctx) return fail(MM_ERR_INVALID, "null context");
  if (!d) return fail(MM_ERR_INVALID, "null matrix pointer");
  if (n == 0) return fail(MM_ERR_INVALID, "matrix dimensions must be positive");
  int rc;
  if ((rc = check_bool_shape("N", n)) != MM_OK) return rc;
  if ((rc = check_batch(batch, n, n, n)) != MM_OK) return rc;
  if ((rc = check_device_alignment(d, d, d)) != MM_OK) return rc;
  if (flags != 0) return fail(MM_ERR_INVALID, "flags is reserved and must be 0");
  std::lock_guard<std::mutex> lock(ctx->mutex);
  MM_CUDA_TRY(cudaSetDevice(ctx->device));
  cudaStream_t s = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : ctx->stream;
  cudaStreamCaptureStatus capture;
  cudaEvent_t *pe;
  if ((rc = begin_call(ctx, s, /*profile=*/true, &capture, &pe)) != MM_OK) return rc;
  if (pe) MM_CUDA_TRY(cudaEventRecord(pe[1], s));  // no preparation: the whole call is main time
  if ((rc = mm::bool_closure(d, n, batch, s)) != MM_OK) return rc;
  if (pe) MM_CUDA_TRY(cudaEventRecord(pe[2], s));
  return MM_OK;
}

int mm_kernel_execute(mm_context *ctx, int dtype, int map_op, int reduce_op, int flags,
                      const void *a, const void *b, void *c, unsigned n, unsigned k, unsigned m,
                      double *seconds_device, double *seconds_wall) {
  return kernel_execute(ctx, dtype, map_op, reduce_op, flags, a, b, c, n, k, m, seconds_device, seconds_wall, nullptr);
}

int mm_context_set_profiling(mm_context *ctx, int enable) {
  if (!ctx) return fail(MM_ERR_INVALID, "null context");
  std::lock_guard<std::mutex> lock(ctx->mutex);
  ctx->profiling = enable != 0;
  ctx->prof_calls = 0;
  return MM_OK;
}

int mm_context_profile_read(mm_context *ctx, double *prep_sum, double *main_sum, int *calls) {
  if (!ctx) return fail(MM_ERR_INVALID, "null context");
  std::lock_guard<std::mutex> lock(ctx->mutex);
  MM_CUDA_TRY(cudaSetDevice(ctx->device));
  double prep = 0.0, main_s = 0.0;
  for (int i = 0; i < ctx->prof_calls; ++i) {
    cudaEvent_t *e = &ctx->prof_events[3 * i];
    MM_CUDA_TRY(cudaEventSynchronize(e[2]));
    float ms_prep = 0.f, ms_main = 0.f;
    MM_CUDA_TRY(cudaEventElapsedTime(&ms_prep, e[0], e[1]));
    MM_CUDA_TRY(cudaEventElapsedTime(&ms_main, e[1], e[2]));
    prep += 1e-3 * ms_prep;
    main_s += 1e-3 * ms_main;
  }
  if (prep_sum) *prep_sum = prep;
  if (main_sum) *main_sum = main_s;
  if (calls) *calls = ctx->prof_calls;
  ctx->prof_calls = 0;
  return MM_OK;
}

int mm_kernel_launch_count(int dtype, int map_op, int reduce_op, int flags) {
  if (!valid_dtype(dtype) || !valid_op(map_op) || !valid_op(reduce_op)) return -1;
  switch (select_path(dtype, map_op, reduce_op, flags, 2, 64)) {
    case kPathTcgen05:
      // B's preparation + [float's second preparation pass, or A's transpose] + GEMM
      return 2 + ((dtype == MM_DTYPE_FLOAT || (flags & MM_FLAG_TRANSPOSED_A)) ? 1 : 0);
    case kPathDmma: return 1;
    case kPathSemiring: return 1;
  }
  return -1;
}

const char *mm_kernel_path(int dtype, int map_op, int reduce_op, int flags) {
  if (!valid_dtype(dtype) || !valid_op(map_op) || !valid_op(reduce_op)) return "invalid";
  switch (select_path(dtype, map_op, reduce_op, flags, 2, 64)) {
    case kPathTcgen05:
      if (dtype == MM_DTYPE_BFLOAT16) return "wgmma_bf16";
      return dtype == MM_DTYPE_FLOAT ? "wgmma_tf32" : (dtype == MM_DTYPE_UINT8 ? "wgmma_i8" : "wgmma_f16");
    case kPathDmma: return "dmma_f64";
    case kPathSemiring: return "semiring_simt";
  }
  return "invalid";
}

int mm_gemm_host(mm_context *ctx, int dtype, int map_op, int reduce_op, int flags, const void *a,
                 const void *b, void *c, unsigned n, unsigned k, unsigned m, double *seconds_device,
                 double *seconds_wall) {
  int rc = check_args(dtype, map_op, reduce_op, a, b, c, n, k, m);
  if (rc != MM_OK) return rc;
  if (!ctx) {
    // the per-process default: one context on $MM_DEVICE, or an mm_multi over $MM_NUM_GPUS devices
    const bool split = env_int("MM_NUM_GPUS", 1) > 1 && !(flags & MM_FLAG_TRANSPOSED_A);
    {
      std::lock_guard<std::mutex> lock(g_default_mutex);
      if (split && !g_default_multi) rc = mm_multi_create(env_int("MM_NUM_GPUS", 1), nullptr, &g_default_multi);
      if (!split && !g_default_ctx) rc = mm_context_create(env_int("MM_DEVICE", 0), &g_default_ctx);
      if (rc != MM_OK) return rc;
    }
    if (split) {
      return mm_multi_gemm_host(g_default_multi, dtype, map_op, reduce_op, flags, a, b, c, n, k, m, seconds_device,
                                seconds_wall);
    }
    ctx = g_default_ctx;
  }
  const auto t0 = std::chrono::high_resolution_clock::now();
  std::lock_guard<std::mutex> lock(ctx->mutex);
  Pipeline p{ctx, dtype, map_op, reduce_op, flags, static_cast<const unsigned char *>(a),
             static_cast<const unsigned char *>(b), static_cast<unsigned char *>(c), n, k, m, mm_dtype_size(dtype),
             select_path(dtype, map_op, reduce_op, flags, n, k)};
  BPlan bp;
  bp.k0 = 0;
  bp.k1 = k;
  rc = p.upload_b(bp);
  if (rc == MM_OK) {
    rc = p.run(bp, seconds_device);
  } else {
    cudaStreamSynchronize(ctx->copy_in);
  }
  if (rc != MM_OK) return rc;
  if (seconds_wall) {
    *seconds_wall = std::chrono::duration<double>(std::chrono::high_resolution_clock::now() - t0).count();
  }
  return MM_OK;
}

// ---- multi-GPU ---------------------------------------------------------------------------------

int mm_multi_create(int n_gpus, const int *devices, mm_multi **out) {
  if (!out) return fail(MM_ERR_INVALID, "null output pointer");
  *out = nullptr;
  if (n_gpus < 1) return fail(MM_ERR_INVALID, "mm_multi_create needs at least one device");
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) {
    return fail(MM_ERR_CUDA, std::string("no CUDA device available: ") +
                                 (e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0"));
  }
  if (!devices && n_gpus > count) {  // an explicit list may name a device more than once (tests do)
    return fail(MM_ERR_INVALID, "mm_multi_create: " + std::to_string(n_gpus) + " devices requested, " +
                                    std::to_string(count) + " visible");
  }
  return create_multi(n_gpus, devices, out);
}

int mm_multi_destroy(mm_multi *mu) {
  if (!mu) return MM_OK;
  for (size_t g = 0; g < mu->ctx.size(); ++g) {
    if (g < mu->parts_dev.size() && mu->parts_dev[g]) {
      cudaSetDevice(mu->ctx[g]->device);
      cudaFree(mu->parts_dev[g]);
    }
  }
  for (mm_context *c : mu->ctx) destroy_context(c);
  delete mu;
  return MM_OK;
}

int mm_multi_device_count(const mm_multi *mu) { return mu ? int(mu->ctx.size()) : 0; }

mm_context *mm_multi_context(mm_multi *mu, int index) {
  if (!mu || index < 0 || index >= int(mu->ctx.size())) return nullptr;
  return mu->ctx[index];
}

int mm_multi_peer_access(const mm_multi *mu) { return (mu && mu->peer) ? 1 : 0; }

int mm_multi_partition(int n_gpus, int index, unsigned n, unsigned k, unsigned *row_begin, unsigned *row_end,
                       unsigned *b_row_begin, unsigned *b_row_end) {
  if (n_gpus < 1 || index < 0 || index >= n_gpus) return fail(MM_ERR_INVALID, "mm_multi_partition: bad device count / index");
  const Partition p = partition_for(n_gpus, index, n, k, /*sliced_b=*/n_gpus > 1);
  if (row_begin) *row_begin = p.r0;
  if (row_end) *row_end = p.r1;
  if (b_row_begin) *b_row_begin = p.k0;
  if (b_row_end) *b_row_end = p.k1;
  return MM_OK;
}

int mm_multi_gemm_host(mm_multi *mu, int dtype, int map_op, int reduce_op, int flags, const void *a, const void *b,
                       void *c, unsigned n, unsigned k, unsigned m, double *seconds_device, double *seconds_wall) {
  if (!mu) return fail(MM_ERR_INVALID, "null multi-GPU context");
  int rc = check_args(dtype, map_op, reduce_op, a, b, c, n, k, m);
  if (rc != MM_OK) return rc;
  const auto t0 = std::chrono::high_resolution_clock::now();
  std::lock_guard<std::mutex> lock(mu->mutex);
  rc = multi_gemm_host_locked(mu, dtype, map_op, reduce_op, flags, a, b, c, n, k, m, seconds_device);
  if (rc != MM_OK) return rc;
  if (seconds_wall) {
    *seconds_wall = std::chrono::duration<double>(std::chrono::high_resolution_clock::now() - t0).count();
  }
  return MM_OK;
}

int mm_multi_upload(mm_multi *mu, int dtype, int flags, const void *a, const void *b, unsigned n, unsigned k,
                    unsigned m) {
  if (!mu) return fail(MM_ERR_INVALID, "null multi-GPU context");
  std::lock_guard<std::mutex> lock(mu->mutex);
  clear_resident(mu);  // a failed upload, rejected arguments included, leaves no resident problem behind
  int rc = check_args(dtype, MM_OP_MULTIPLY, MM_OP_ADD, a, b, a /*non-null placeholder*/, n, k, m);
  if (rc != MM_OK) return rc;
  if (flags & MM_FLAG_TRANSPOSED_A) {
    return fail(MM_ERR_UNSUPPORTED, "the row-block split over GPUs needs row-major A (MM_TRANSPOSED_A is set)");
  }
  const int G = int(mu->ctx.size());
  const size_t es = mm_dtype_size(dtype);
  std::vector<uint64_t> gen(G, 0);
  HostBarrier barrier(G);
  rc = fan_out(G, [&](int g) -> int {
    mm_context *ctx = mu->ctx[g];
    std::lock_guard<std::mutex> ctx_lock(ctx->mutex);
    gen[g] = ++ctx->staging_gen;
    const Partition part = partition_for(G, g, n, k, mu->peer);
    const unsigned r0 = part.r0, r1 = part.r1, part_rows = part.part_rows;
    const unsigned rows = std::max(1u, r1 - r0);
    auto body = [&]() -> int {
      MM_CUDA_TRY(cudaSetDevice(ctx->device));
      int r;
      if ((r = ensure(ctx, ctx->staging[0], size_t(rows) * k * es, false)) != MM_OK) return r;
      if ((r = ensure(ctx, ctx->staging[1], size_t(k) * m * es, false)) != MM_OK) return r;
      if ((r = ensure(ctx, ctx->staging[2], size_t(rows) * m * es, false)) != MM_OK) return r;
      unsigned char *db = static_cast<unsigned char *>(ctx->staging[1].ptr);
      const unsigned k0 = part.k0, k1 = part.k1;
      const size_t off = size_t(k0) * m * es;
      if (k1 > k0) {
        MM_CUDA_TRY(cudaMemcpyAsync(db + off, static_cast<const unsigned char *>(b) + off, size_t(k1 - k0) * m * es,
                                    cudaMemcpyHostToDevice, ctx->copy_in));
      }
      MM_CUDA_TRY(cudaEventRecord(ctx->ev_slice, ctx->copy_in));
      if (r1 > r0) {
        MM_CUDA_TRY(cudaMemcpyAsync(ctx->staging[0].ptr, static_cast<const unsigned char *>(a) + size_t(r0) * k * es,
                                    size_t(r1 - r0) * k * es, cudaMemcpyHostToDevice, ctx->copy_in));
      }
      return MM_OK;
    };
    const int rc1 = body();
    barrier.arrive_and_wait();
    int rc2 = MM_OK;
    if (rc1 == MM_OK && mu->peer) {
      rc2 = refresh_parts(mu, g);
    }
    barrier.arrive_and_wait();
    if (rc1 == MM_OK && rc2 == MM_OK && mu->peer) {
      auto gather = [&]() -> int {
        MM_CUDA_TRY(cudaStreamWaitEvent(ctx->stream, ctx->ev_slice, 0));
        for (int j = 0; j < G; ++j) {
          if (j != g) MM_CUDA_TRY(cudaStreamWaitEvent(ctx->stream, mu->ctx[j]->ev_slice, 0));
        }
        return mm::gather_b_rows(mu->parts_dev[g], part_rows, ctx->staging[1].ptr, es, k, m, ctx->stream);
      };
      rc2 = gather();
    }
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->copy_in);
    cudaStreamSynchronize(ctx->stream);
    barrier.arrive_and_wait();
    return rc1 != MM_OK ? rc1 : rc2;
  });
  if (rc != MM_OK) return rc;
  mu->n = n;
  mu->k = k;
  mu->m = m;
  mu->dtype = dtype;
  mu->gen = gen;
  return MM_OK;
}

int mm_multi_execute(mm_multi *mu, int dtype, int map_op, int reduce_op, int flags, unsigned n, unsigned k, unsigned m,
                     double *seconds_device, double *seconds_wall) {
  if (!mu) return fail(MM_ERR_INVALID, "null multi-GPU context");
  if (!valid_dtype(dtype) || !valid_op(map_op) || !valid_op(reduce_op)) return fail(MM_ERR_INVALID, "unknown type / operator code");
  std::lock_guard<std::mutex> lock(mu->mutex);
  int rc = check_resident(mu, "mm_multi_execute", dtype, n, k, m);
  if (rc != MM_OK) return rc;
  mu->executed = false;  // C is rewritten below: a failed execute leaves nothing to download
  const int G = int(mu->ctx.size());
  std::vector<double> dev_s(G, 0.0);
  const auto t0 = std::chrono::high_resolution_clock::now();
  HostBarrier barrier(G);
  FitsAgreement fits(barrier, G);
  rc = fan_out(G, [&](int g) -> int {
    const Partition part = partition_for(G, g, n, k, mu->peer);
    const unsigned r0 = part.r0, r1 = part.r1;
    int r = MM_OK;
    if (r1 > r0) {
      mm_context *ctx = mu->ctx[g];
      const mm::AgreeFn agree = fits.agree(g);
      r = kernel_execute(ctx, dtype, map_op, reduce_op, flags, ctx->staging[0].ptr, ctx->staging[1].ptr,
                         ctx->staging[2].ptr, r1 - r0, k, m, &dev_s[g], nullptr, &agree);
    }
    fits.finish(g);
    return r;
  });
  if (rc != MM_OK) return rc;
  mu->executed = true;
  if (seconds_device) *seconds_device = *std::max_element(dev_s.begin(), dev_s.end());
  if (seconds_wall) {
    *seconds_wall = std::chrono::duration<double>(std::chrono::high_resolution_clock::now() - t0).count();
  }
  return MM_OK;
}

int mm_multi_download(mm_multi *mu, int dtype, void *c, unsigned n, unsigned m) {
  if (!mu || !c) return fail(MM_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lock(mu->mutex);
  const int rc = check_resident(mu, "mm_multi_download", dtype, n, mu->k, m);
  if (rc != MM_OK) return rc;
  if (!mu->executed) return fail(MM_ERR_INVALID, "mm_multi_download: no mm_multi_execute since the last upload");
  const int G = int(mu->ctx.size());
  const size_t es = mm_dtype_size(dtype);
  return fan_out(G, [&](int g) -> int {
    const Partition part = partition_for(G, g, n, 64, false);
    const unsigned r0 = part.r0, r1 = part.r1;
    if (r1 == r0) return MM_OK;
    mm_context *ctx = mu->ctx[g];
    return mm_copy_to_host(ctx, static_cast<unsigned char *>(c) + size_t(r0) * m * es, ctx->staging[2].ptr,
                           size_t(r1 - r0) * m * es);
  });
}

}  // extern "C"
