// Tensor-core path of the hot path for the dense (Multiply, Add) contraction on float, half, bfloat16 and uint8_t:
//   C[N x M] = A[N x K] * B[K x M]
// sm_90a counterpart of the reference's PE chain + streamers (kernel/Compute.cpp:53-146,
// kernel/Memory.cpp:58-438) for MM_MAP_OP=Multiply, MM_REDUCE_OP=Add, MM_DATA_TYPE in {float, half, uint8_t}
// (uint8_t: wgmma u8 x u8 with exact 32-bit integer accumulation, truncated to 8 bits in the epilogue = the
// reference's arithmetic modulo 256, bit for bit; reference CMakeLists.txt:43-46).
//
// Structure (one persistent CTA per SM, warp-specialised, no CUTLASS):
//   warpgroup 0    TMA producer (the role of ReadA / ReadB / FeedB): one thread issues cp.async.bulk.tensor
//                  of 128-byte-swizzled A (128 x BK) and B (BN x BK) tiles, both K-major, into a
//                  STAGES-deep shared-memory ring with mbarrier full/empty pairs.
//   warpgroups 1-2 consumers (the PE chain + WriteC, kernel/Memory.cpp:361-392): each issues wgmma
//                  (M = 64, N = BN, K = 32 bytes) for its 64 rows of the 128-row tile into FP32 (S32)
//                  register accumulators, releases ring stages as their wgmma groups retire, then
//                  converts and writes its rows of C: per warp 16 x 32 blocks staged in swizzled shared
//                  memory and written with TMA stores (clipped to n < N, m < M by the tensor map), or
//                  direct stores.  The producer keeps fetching the next tile meanwhile.
//   cta_group = 2  a cluster of two CTAs computes a 256 x BN tile: each CTA loads its own 128 rows of A
//                  and HALF of the B tile, multicast into both CTAs, so B's L2 -> SM traffic halves.
//
// wgmma reads 32-bit (tf32) and 8-bit operands only K-major, so B is always consumed from a transposed
// K-major copy (M x K), made by the operand preparation below.
//
// Operand preparation (O(N*K + K*M) bytes against O(N*K*M) flops):
//   * tf32 wgmma reads only the upper 19 bits of each fp32 operand, i.e. it TRUNCATES.  The
//     reference's inputs are all positive (U[1,10], test/TestSimulation.cpp:46-55), so truncation
//     would bias every product by about -2^-11 * 2 and land the sum right at the 1e-3 tolerance.
//     A and B are therefore rounded to nearest TF32 (cvt.rna.tf32.f32) into scratch copies first.
//   * half, bfloat16 and uint8_t A are K-major as stored; B is transposed.  bfloat16 moves the same bits as
//     half, so it shares half's transpose kernel.
//   * A value rounded to TF32 keeps 10 mantissa bits, as many as a half has.  So the same passes also write the
//     rounded operands as halves and note, per distinct operand, whether every value is 0 or a normal half
//     (fits_half.h).  A problem whose A and B both fit runs on the f16 wgmma, which multiplies the very same values
//     at twice the TF32 issue rate (gemm_wgmma.cuh); any other problem stays on TF32.
//
// The GEMM kernel and its launcher are in gemm_wgmma.cuh.  This unit instantiates them for tf32, f16 and
// u8; the bf16 instantiations are in gemm_wgmma_bf16.cu, the accumulate kernels in gemm_wgmma_acc.cu.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "fits_half.h"
#include "gemm_wgmma.cuh"
#include "ptx_sm90.cuh"
#include "tma_host.cuh"

namespace mm {
namespace {

// Round to nearest TF32, ties away from zero.  cvt.rna rounds every finite |x| >= 0x7F7FF000 up to
// infinity; a finite operand must stay finite (x * 0.5 is finite), so those saturate to the largest
// finite TF32 value, +-0x7F7FE000.  Infinities and NaN pass through.
__device__ __forceinline__ float round_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  const bool overflowed = (r & 0x7FFFFFFFu) == 0x7F800000u && (__float_as_uint(x) & 0x7FFFFFFFu) != 0x7F800000u;
  return __uint_as_float(overflowed ? ((r & 0x80000000u) | 0x7F7FE000u) : r);
}

// ---- operand preparation ------------------------------------------------------------------------

__device__ __forceinline__ uint32_t half2_bits(float lo, float hi) {
  const __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<const uint32_t *>(&h);
}

// dst[i] = rna_tf32(src[i]); count4 float4 per problem, blockIdx.y = problem of a batch (packed).  HALF: dst16 gets the
// same values as halves, and fits[problem] is cleared when one of them is not exactly a half (one store per block).
template <bool HALF>
__global__ void __launch_bounds__(256)
round_tf32_kernel(const float4 *__restrict__ src, float4 *__restrict__ dst, size_t count4, uint2 *__restrict__ dst16,
                  unsigned int *__restrict__ fits) {
  src += size_t(blockIdx.y) * count4;
  dst += size_t(blockIdx.y) * count4;
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  bool fit = true;
  for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < count4; i += stride) {
    float4 v = src[i];
    v.x = round_tf32(v.x);
    v.y = round_tf32(v.y);
    v.z = round_tf32(v.z);
    v.w = round_tf32(v.w);
    dst[i] = v;
    if constexpr (HALF) {
      dst16[size_t(blockIdx.y) * count4 + i] = make_uint2(half2_bits(v.x, v.y), half2_bits(v.z, v.w));
      fit = fit && tf32_fits_half(__float_as_uint(v.x)) && tf32_fits_half(__float_as_uint(v.y)) &&
            tf32_fits_half(__float_as_uint(v.z)) && tf32_fits_half(__float_as_uint(v.w));
    }
  }
  if constexpr (HALF) {
    if (__syncthreads_or(!fit) && threadIdx.x == 0) fits[blockIdx.y] = 0u;
  }
}

// B (row-major K x M, 16-byte vectors) -> dst (same layout), panel by panel: a work item is
// PANEL_ROWS k-rows of one panel of `panel_v` vectors per row; items are numbered panel-major and
// dealt round-robin to the CTAs of a persistent grid, so panels complete in ascending order.  Each
// finished item bumps ready[panel] (release pattern: every thread fences its stores, the CTA syncs,
// one thread adds).  ROUND: elements are floats rounded to nearest TF32; otherwise a plain copy.
// `parts` non-null: k-row r is read from parts[r / part_rows] — full-size K x M arrays on (peer) GPUs
// of which only that slice of rows is valid; rows whose source IS the destination are skipped.
constexpr int PREP_THREADS = 512;
constexpr int PREP_WARPS = PREP_THREADS / 32;
constexpr int PANEL_ROWS = 64;
constexpr int PANEL_ROW_SLOTS = PANEL_ROWS / PREP_WARPS;  // rows per warp per item (4)

template <bool ROUND>
__device__ __forceinline__ uint4 prep_vec(uint4 v) {
  if (ROUND) {
    v.x = __float_as_uint(round_tf32(__uint_as_float(v.x)));
    v.y = __float_as_uint(round_tf32(__uint_as_float(v.y)));
    v.z = __float_as_uint(round_tf32(__uint_as_float(v.z)));
    v.w = __float_as_uint(round_tf32(__uint_as_float(v.w)));
  }
  return v;
}

template <bool ROUND>
__global__ void __launch_bounds__(PREP_THREADS)
prep_b_panels_kernel(const uint4 *__restrict__ single, const uint4 *const *__restrict__ parts, uint32_t part_rows,
                     uint4 *__restrict__ dst, uint32_t k, uint32_t row_v, uint32_t panel_v,
                     unsigned int *__restrict__ ready) {
  const uint32_t warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const uint32_t panels = (row_v + panel_v - 1) / panel_v;
  const uint32_t items_per_panel = (k + PANEL_ROWS - 1) / PANEL_ROWS;
  const uint32_t items = panels * items_per_panel;
  for (uint32_t item = blockIdx.x; item < items; item += gridDim.x) {
    const uint32_t panel = item / items_per_panel;
    const uint32_t r0 = (item - panel * items_per_panel) * PANEL_ROWS;
    const uint32_t v0 = panel * panel_v;
    const uint32_t w = min(panel_v, row_v - v0);
    for (uint32_t c0 = 0; c0 < w; c0 += 64) {   // 64 vectors (1 KiB) of a row per pass: 8 loads in flight per thread
      uint4 buf[PANEL_ROW_SLOTS][2];
      bool live[PANEL_ROW_SLOTS][2];
#pragma unroll
      for (int u = 0; u < PANEL_ROW_SLOTS; ++u) {
        const uint32_t r = r0 + warp + u * PREP_WARPS;
        const uint4 *src = single;
        if (parts != nullptr && r < k) src = parts[r / part_rows];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint32_t c = c0 + lane + 32 * h;
          const size_t off = size_t(r) * row_v + v0 + c;
          live[u][h] = (r < k) && (c < w) && (src + off != static_cast<const uint4 *>(dst) + off);
          if (live[u][h]) buf[u][h] = src[off];
        }
      }
#pragma unroll
      for (int u = 0; u < PANEL_ROW_SLOTS; ++u) {
        const uint32_t r = r0 + warp + u * PREP_WARPS;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint32_t c = c0 + lane + 32 * h;
          if (live[u][h]) dst[size_t(r) * row_v + v0 + c] = prep_vec<ROUND>(buf[u][h]);
        }
      }
    }
    if (ready != nullptr) {
      __threadfence();
      __syncthreads();
      if (threadIdx.x == 0) atomicAdd(ready + panel, 1u);
    }
  }
}

template <typename T, bool ROUND>
__device__ __forceinline__ T prep_value(T x) {
  return x;
}
template <>
__device__ __forceinline__ float prep_value<float, true>(float x) {
  return round_tf32(x);
}

// dst[c][r] = f(src[r][c]) for src of shape src_rows x src_cols (row-major): 64 x 64 tiles through
// shared memory so that both the reads and the writes are row-contiguous.  blockIdx.z = problem of a
// batch: packed sources, packed destinations.  ROUND (float to TF32): dst16 gets the rounded values as halves too, and
// fits[problem] is cleared when one of them is not exactly a half, as in round_tf32_kernel.
template <typename T, bool ROUND>
__global__ void __launch_bounds__(256)
transpose_prep_kernel(const T *__restrict__ src, T *__restrict__ dst, uint32_t src_rows,
                      uint32_t src_cols, __half *__restrict__ dst16, unsigned int *__restrict__ fits) {
  constexpr int TILE = 64;
  constexpr int PAD = (sizeof(T) >= 4) ? 1 : 2;
  __shared__ T tile[TILE][TILE + PAD];
  src += size_t(blockIdx.z) * src_rows * src_cols;
  dst += size_t(blockIdx.z) * src_rows * src_cols;
  const uint32_t c0 = blockIdx.x * TILE;
  const uint32_t r0 = blockIdx.y * TILE;
  const int x = threadIdx.x % TILE;
  const int y = threadIdx.x / TILE;  // 0..3
#pragma unroll 4
  for (int i = y; i < TILE; i += 4) {
    const uint32_t r = r0 + i, c = c0 + x;
    if (r < src_rows && c < src_cols) tile[i][x] = prep_value<T, ROUND>(src[size_t(r) * src_cols + c]);
  }
  __syncthreads();
  bool fit = true;
#pragma unroll 4
  for (int i = y; i < TILE; i += 4) {
    const uint32_t c = c0 + i, r = r0 + x;  // dst row = src col
    if (c < src_cols && r < src_rows) {
      const T v = tile[x][i];
      dst[size_t(c) * src_rows + r] = v;
      if constexpr (ROUND) {
        dst16[size_t(blockIdx.z) * src_rows * src_cols + size_t(c) * src_rows + r] = __float2half_rn(v);
        fit = fit && tf32_fits_half(__float_as_uint(v));
      }
    }
  }
  if constexpr (ROUND) {
    if (__syncthreads_or(!fit) && threadIdx.x == 0) fits[blockIdx.z] = 0u;
  }
}

// ---- 3xTF32 operand construction (MM_FLAG_TF32X3) ------------------------------------------------
// x = hi + lo with hi = rna_tf32(x), lo = rna_tf32(x - hi).  A*B ~= hi_a*hi_b + hi_a*lo_b + lo_a*hi_b
// (the dropped lo*lo term is 2^-22 relative).  The three products are folded into ONE GEMM with
// K' = 3K by interleaving 16-element k-blocks:  A' = [hi | hi | lo],  B'^T = [hi | lo | hi],
// so the unchanged wgmma kernel accumulates all three in its FP32 register accumulators.
// Infinities: lo = 0 (inf - inf would be NaN), and the hi that meets the other operand's lo (A's second
// block, B's third) carries 0 in place of +-inf (inf * 0 would be NaN where the other operand is exactly
// TF32).  Only hi * hi carries infinities, so C gets IEEE's +-inf; NaN still propagates through hi.
constexpr int SPLIT_BLOCK = 16;  // K % 16 == 0 by the reference's shape rule for float

__device__ __forceinline__ void split_tf32(float x, float &hi, float &lo) {
  hi = round_tf32(x);
  lo = isinf(x) ? 0.0f : round_tf32(x - hi);
}

// hi for the cross terms: +-inf -> 0
__device__ __forceinline__ float finite_or_zero(float hi) { return isinf(hi) ? 0.0f : hi; }

// dst[r][3K]: per 16-block of k -> [hi16 | hi16 | lo16]; one thread per float4 of the source row.
__global__ void __launch_bounds__(256)
split3_rows_kernel(const float4 *__restrict__ src, float4 *__restrict__ dst, size_t rows, uint32_t k) {
  const size_t k4 = k / 4;
  const size_t total = rows * k4;
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const size_t r = i / k4;
    const uint32_t c4 = uint32_t(i - r * k4);       // float4 index within the row
    const uint32_t blk = c4 / (SPLIT_BLOCK / 4), in = c4 % (SPLIT_BLOCK / 4);
    const float4 v = src[i];
    float4 hi, lo;
    split_tf32(v.x, hi.x, lo.x);
    split_tf32(v.y, hi.y, lo.y);
    split_tf32(v.z, hi.z, lo.z);
    split_tf32(v.w, hi.w, lo.w);
    float4 *row = dst + r * (3 * k4) + size_t(blk) * (3 * SPLIT_BLOCK / 4) + in;
    row[0] = hi;
    row[SPLIT_BLOCK / 4] = make_float4(finite_or_zero(hi.x), finite_or_zero(hi.y), finite_or_zero(hi.z),
                                       finite_or_zero(hi.w));
    row[2 * SPLIT_BLOCK / 4] = lo;
  }
}

// src (src_rows = K) x (src_cols) row-major -> dst[c][3K] with per-16-block [a | b | c] where
// B_ORDER selects (hi, lo, hi') for the B operand and (hi, hi', lo) for a transposed A, hi' =
// finite_or_zero(hi).  blockIdx.z =
// problem of a batch, as in transpose_prep_kernel.
template <bool B_ORDER>
__global__ void __launch_bounds__(256)
split3_transpose_kernel(const float *__restrict__ src, float *__restrict__ dst, uint32_t src_rows,
                        uint32_t src_cols) {
  constexpr int TILE = 64;
  __shared__ float tile[TILE][TILE + 1];
  src += size_t(blockIdx.z) * src_rows * src_cols;
  dst += size_t(blockIdx.z) * src_rows * src_cols * 3;
  const uint32_t c0 = blockIdx.x * TILE;
  const uint32_t r0 = blockIdx.y * TILE;
  const int x = threadIdx.x % TILE;
  const int y = threadIdx.x / TILE;
#pragma unroll 4
  for (int i = y; i < TILE; i += 4) {
    const uint32_t r = r0 + i, c = c0 + x;
    if (r < src_rows && c < src_cols) tile[i][x] = src[size_t(r) * src_cols + c];
  }
  __syncthreads();
#pragma unroll 4
  for (int i = y; i < TILE; i += 4) {
    const uint32_t c = c0 + i, r = r0 + x;  // dst row = src col; r = k index
    if (c < src_cols && r < src_rows) {
      float hi, lo;
      split_tf32(tile[x][i], hi, lo);
      float *out = dst + size_t(c) * (3 * size_t(src_rows)) + size_t(r / SPLIT_BLOCK) * (3 * SPLIT_BLOCK) +
                   (r % SPLIT_BLOCK);
      out[0] = hi;
      out[SPLIT_BLOCK] = B_ORDER ? lo : finite_or_zero(hi);
      out[2 * SPLIT_BLOCK] = B_ORDER ? finite_or_zero(hi) : lo;
    }
  }
}

// ---- host side -----------------------------------------------------------------------------------

size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

template <typename T, bool ROUND>
void launch_transpose(const void *src, void *dst, uint32_t src_rows, uint32_t src_cols, cudaStream_t stream,
                      unsigned copies, void *dst16 = nullptr, unsigned int *fits = nullptr) {
  dim3 grid((src_cols + 63) / 64, (src_rows + 63) / 64, copies);
  transpose_prep_kernel<T, ROUND><<<grid, 256, 0, stream>>>(static_cast<const T *>(src), static_cast<T *>(dst),
                                                           src_rows, src_cols, static_cast<__half *>(dst16), fits);
}

// Rounds `copies` packed problems of count4 float4 each; with `dst16` the fp16 copies and fits flags too.
int launch_round(const void *src, void *dst, size_t count4, unsigned copies, void *dst16, unsigned int *fits,
                 cudaStream_t stream) {
  const int blocks = int(std::min<size_t>((count4 + 255) / 256, size_t(num_sms()) * 16));
  const dim3 grid(std::max(blocks, 1), copies);
  const float4 *s = static_cast<const float4 *>(src);
  float4 *d = static_cast<float4 *>(dst);
  if (dst16 != nullptr) {
    // see tcgen05_prepare_b
    MM_CUDA_TRY(cudaFuncSetAttribute(round_tf32_kernel<true>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                     cudaSharedmemCarveoutMaxShared));
    round_tf32_kernel<true><<<grid, 256, 0, stream>>>(s, d, count4, static_cast<uint2 *>(dst16), fits);
  } else {
    MM_CUDA_TRY(cudaFuncSetAttribute(round_tf32_kernel<false>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                     cudaSharedmemCarveoutMaxShared));
    round_tf32_kernel<false><<<grid, 256, 0, stream>>>(s, d, count4, nullptr, nullptr);
  }
  return MM_OK;
}

bool split3(int dtype, int flags) { return dtype == MM_DTYPE_FLOAT && (flags & MM_FLAG_TF32X3); }

int launch_panels(bool round, const BSource &src, void *dst, size_t elem_bytes, unsigned k, unsigned m,
                  unsigned panel_cols, unsigned int *ready, int grid, cudaStream_t stream) {
  const uint32_t row_v = uint32_t(size_t(m) * elem_bytes / 16);
  const uint32_t panel_v = uint32_t(size_t(panel_cols) * elem_bytes / 16);
  const uint4 *single = static_cast<const uint4 *>(src.b);
  const uint4 *const *parts = reinterpret_cast<const uint4 *const *>(src.src);
  if (round) {
    prep_b_panels_kernel<true><<<grid, PREP_THREADS, 0, stream>>>(single, parts, src.part_rows, static_cast<uint4 *>(dst),
                                                                 k, row_v, panel_v, ready);
  } else {
    prep_b_panels_kernel<false><<<grid, PREP_THREADS, 0, stream>>>(single, parts, src.part_rows, static_cast<uint4 *>(dst),
                                                                  k, row_v, panel_v, ready);
  }
  MM_CUDA_TRY(cudaGetLastError());
  return MM_OK;
}

}  // namespace

// Tail of the scratch: [panel counters of B's preparation, 64 KiB][soft wave-barrier counter, 256 B]
constexpr size_t TILE_SYNC_BYTES = 256;
constexpr size_t B_READY_BYTES = 64 * 1024;  // 16384 panels of >= 128 columns
constexpr size_t TAIL_BYTES = TILE_SYNC_BYTES + B_READY_BYTES;
static_assert(TAIL_BYTES == kTcgen05TailBytes, "common.cuh and gemm_tcgen05.cu disagree on the scratch tail");

Tcgen05Counters tcgen05_counters(void *scratch, size_t scratch_bytes) {
  unsigned char *tail = static_cast<unsigned char *>(scratch) + scratch_bytes;
  return Tcgen05Counters{reinterpret_cast<unsigned int *>(tail - TILE_SYNC_BYTES),
                         reinterpret_cast<unsigned int *>(tail - TAIL_BYTES)};
}

// wgmma reads tf32 and 8-bit operands only K-major; every type takes the K-major copy of B.
bool tcgen05_b_mn(int, int, const Tuning &) { return false; }

bool tcgen05_b_in_place(int dtype, int flags, const Tuning &t) {
  return tcgen05_b_mn(dtype, flags, t) && (dtype == MM_DTYPE_HALF || dtype == MM_DTYPE_UINT8 || t.tf32_no_round());
}

// float on the default TF32 datapath: the preparation also writes fp16 copies and fits flags (HalfScratch)
bool half_copies(int dtype, int flags, const Tuning &t) {
  return dtype == MM_DTYPE_FLOAT && !split3(dtype, flags) && !t.tf32_no_round();
}

size_t b_copy_bytes(int dtype, unsigned k, unsigned m, int flags, unsigned b_copies) {
  return align_up(size_t(b_copies) * m * k * elem_bytes(dtype) * (split3(dtype, flags) ? 3 : 1), 1024);
}
size_t a_copy_bytes(int dtype, unsigned n, unsigned k, int flags, unsigned a_copies) {
  if (dtype != MM_DTYPE_FLOAT && !(flags & MM_FLAG_TRANSPOSED_A)) return 0;
  return align_up(size_t(a_copies) * n * k * elem_bytes(dtype) * (split3(dtype, flags) ? 3 : 1), 1024);
}
size_t fits_bytes(const GemmBatch &batch) {
  return align_up(size_t(batch.a_copies() + batch.b_copies()) * sizeof(unsigned int), 1024);
}

size_t tcgen05_bt_bytes(int dtype, unsigned k, unsigned m, int flags, const Tuning &t, unsigned b_copies) {
  if (tcgen05_b_in_place(dtype, flags, t)) return 0;
  const size_t fp16 = half_copies(dtype, flags, t) ? align_up(size_t(b_copies) * m * k * 2, 1024) : 0;
  return b_copy_bytes(dtype, k, m, flags, b_copies) + fp16;  // [B copy][B fp16]
}

size_t tcgen05_scratch_bytes(int dtype, unsigned n, unsigned k, unsigned m, int flags, const Tuning &t,
                             const GemmBatch &batch) {
  size_t bytes = TAIL_BYTES + tcgen05_bt_bytes(dtype, k, m, flags, t, batch.b_copies());  // counters (tail) + B copies
  bytes += a_copy_bytes(dtype, n, k, flags, batch.a_copies());
  if (half_copies(dtype, flags, t)) bytes += align_up(size_t(batch.a_copies()) * n * k * 2, 1024) + fits_bytes(batch);
  return bytes;
}

HalfScratch tcgen05_half_scratch(void *scratch, size_t scratch_bytes, int dtype, unsigned n, unsigned k, unsigned m,
                                 int flags, const Tuning &t, const GemmBatch &batch) {
  HalfScratch h;
  if (!half_copies(dtype, flags, t)) return h;
  unsigned char *sp = static_cast<unsigned char *>(scratch);
  const size_t bt = tcgen05_bt_bytes(dtype, k, m, flags, t, batch.b_copies());
  h.b = sp + b_copy_bytes(dtype, k, m, flags, batch.b_copies());
  h.a = sp + bt + a_copy_bytes(dtype, n, k, flags, batch.a_copies());
  h.flag_bytes = fits_bytes(batch);
  h.fits_b = reinterpret_cast<unsigned int *>(sp + scratch_bytes - TAIL_BYTES - h.flag_bytes);
  h.fits_a = h.fits_b + batch.b_copies();
  return h;
}

// Copy row-sliced B (slices on peer GPUs) into one local array: the NVLink all-gather of the
// multi-GPU path for the kernel families that consume B as stored.
int gather_b_rows(const BSource &src, void *dst, size_t elem_bytes, unsigned k, unsigned m, cudaStream_t stream) {
  return launch_panels(false, src, dst, elem_bytes, k, m, /*panel_cols=*/unsigned(1024 / elem_bytes), nullptr,
                       num_sms() * 2, stream);
}

int tcgen05_prepare_b(int dtype, const BSource &src, void *bt, unsigned k, unsigned m, int flags, const Tuning &t,
                      const void **b_op, unsigned int *ready, unsigned *ready_target, cudaStream_t stream,
                      unsigned copies, void *bt16, unsigned int *fits) {
  *b_op = bt;
  if (ready_target) *ready_target = 0;
  const bool parts = src.src != nullptr;
  const size_t eb = elem_bytes(dtype);
  if (tcgen05_b_mn(dtype, flags, t)) {
    if (copies != 1) return fail(MM_ERR_UNSUPPORTED, "batched calls need the K-major B copy");
    const bool in_place = tcgen05_b_in_place(dtype, flags, t);
    if (in_place && !parts) {
      *b_op = src.b;  // nothing to prepare
      return MM_OK;
    }
    // float: rounded copy (same layout).  half / unrounded float with slices: plain gather into `bt`.
    if (!in_place && !parts && ready == nullptr) {
      // one local array, nobody waiting on panels: the flat elementwise pass (6.3 TB/s against the panel
      // kernel's 5.1 on a 512 MiB block — the panel order costs row-segment locality)
      const int rc = launch_round(src.b, bt, size_t(k) * m / 4, 1, nullptr, nullptr, stream);
      if (rc != MM_OK) return rc;
      MM_CUDA_TRY(cudaGetLastError());
      return MM_OK;
    }
    const unsigned panel_cols = unsigned(t.block_n());
    const unsigned panels = ceil_div(m, panel_cols);
    const bool publish = ready != nullptr && panels <= B_READY_BYTES / sizeof(unsigned int);
    if (publish && ready_target) *ready_target = ceil_div(k, PANEL_ROWS);
    // co-resident persistent grid (one 512-thread CTA per SM next to the GEMM's CTA) when the GEMM
    // consumes panels while this runs; a wider grid when it runs alone in stream order
    const int grid = publish ? num_sms() : num_sms() * 2;
    // An SM changes its L1 / shared-memory split only when it is idle.  This kernel uses no shared memory; were it
    // to run under the default (L1-heavy) split, the GEMM's CTAs (214 KiB of shared memory) could not become
    // resident next to it and would wait for it to END — measured: the "overlapped" GEMM took exactly its own time
    // plus this kernel's.  Ask for the shared-memory-heavy split so that both fit on an SM together.
    // (Function attributes are per device: set on every call, it is cheap.  A's rounding kernel may share SMs with
    // this one, so it asks for the same split — tcgen05_prepare_a.)
    MM_CUDA_TRY(cudaFuncSetAttribute(prep_b_panels_kernel<true>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                     cudaSharedmemCarveoutMaxShared));
    MM_CUDA_TRY(cudaFuncSetAttribute(prep_b_panels_kernel<false>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                     cudaSharedmemCarveoutMaxShared));
    return launch_panels(!in_place, src, bt, eb, k, m, panel_cols, publish ? ready : nullptr, grid, stream);
  }
  // K-major copy B^T (M x K): tuning knob b_mn = 0, and always for the 3xTF32 split
  const void *b = src.b;
  if (parts) return fail(MM_ERR_UNSUPPORTED, "row-sliced B needs the MN-major B path (gather it first)");
  if (split3(dtype, flags)) {
    dim3 grid((m + 63) / 64, (k + 63) / 64, copies);
    split3_transpose_kernel<true><<<grid, 256, 0, stream>>>(static_cast<const float *>(b), static_cast<float *>(bt), k, m);
  } else if (dtype == MM_DTYPE_FLOAT) {
    if (t.tf32_no_round()) {
      launch_transpose<float, false>(b, bt, k, m, stream, copies);
    } else {
      launch_transpose<float, true>(b, bt, k, m, stream, copies, bt16, fits);
    }
  } else if (dtype == MM_DTYPE_UINT8) {
    launch_transpose<unsigned char, false>(b, bt, k, m, stream, copies);
  } else {
    launch_transpose<__half, false>(b, bt, k, m, stream, copies);
  }
  MM_CUDA_TRY(cudaGetLastError());
  return MM_OK;
}

// `rows` rows of A -> the K-major A operand.  Row-major float A is rounded into `aprep`; row-major
// half, bfloat16 and uint8_t A are used in place; A stored K x N (`transposed`, leading dimension = rows, only whole
// matrices) is transposed into `aprep`.  *a_op receives the operand pointer.  `copies` packed problems:
// the row-wise passes run over copies * rows rows, the transposes take the problem from blockIdx.z.
int tcgen05_prepare_a(int dtype, const void *a, void *aprep, unsigned rows, unsigned k, int flags, const Tuning &t,
                      const void **a_op, cudaStream_t stream, unsigned copies, void *aprep16, unsigned int *fits) {
  const bool transposed = (flags & MM_FLAG_TRANSPOSED_A) != 0;
  const size_t all_rows = size_t(copies) * rows;
  *a_op = a;
  if (split3(dtype, flags)) {
    if (transposed) {
      dim3 grid((rows + 63) / 64, (k + 63) / 64, copies);
      split3_transpose_kernel<false><<<grid, 256, 0, stream>>>(static_cast<const float *>(a),
                                                              static_cast<float *>(aprep), k, rows);
    } else {
      const size_t total4 = all_rows * k / 4;
      const int blocks = int(std::min<size_t>((total4 + 255) / 256, size_t(num_sms()) * 16));
      split3_rows_kernel<<<blocks, 256, 0, stream>>>(static_cast<const float4 *>(a),
                                                    static_cast<float4 *>(aprep), all_rows, k);
    }
    *a_op = aprep;
  } else if (dtype == MM_DTYPE_FLOAT) {
    if (transposed) {
      if (t.tf32_no_round()) {
        launch_transpose<float, false>(a, aprep, k, rows, stream, copies);
      } else {
        launch_transpose<float, true>(a, aprep, k, rows, stream, copies, aprep16, fits);  // A stored K x N -> N x K
      }
      *a_op = aprep;
    } else if (!t.tf32_no_round()) {
      const int rc = launch_round(a, aprep, size_t(rows) * k / 4, copies, aprep16, fits, stream);
      if (rc != MM_OK) return rc;
      *a_op = aprep;
    }
  } else if (transposed) {
    if (dtype == MM_DTYPE_UINT8) launch_transpose<unsigned char, false>(a, aprep, k, rows, stream, copies);
    else launch_transpose<__half, false>(a, aprep, k, rows, stream, copies);
    *a_op = aprep;
  }
  MM_CUDA_TRY(cudaGetLastError());
  return MM_OK;
}

namespace {
int gemm_dispatch(int dtype, const void *a_op, const void *b_op, void *c, unsigned rows, unsigned k, unsigned m,
                  int flags, const Tuning &t, unsigned int *tile_sync, const unsigned int *b_ready,
                  unsigned b_ready_target, bool attributes_only, cudaStream_t stream, const GemmBatch &batch,
                  bool accumulate = false, const HalfOperands &half = HalfOperands{}) {
  if (accumulate) {
    if (split3(dtype, flags)) k *= 3;
    return wgmma_accumulate_gemm(dtype, a_op, b_op, c, rows, k, m, t, tile_sync, b_ready, b_ready_target,
                                 attributes_only, stream, batch, half);
  }
  if (dtype == MM_DTYPE_BFLOAT16) {
    return wgmma_bf16_gemm(a_op, b_op, c, rows, k, m, t, tile_sync, b_ready, b_ready_target, attributes_only, stream,
                           batch);
  }
  if (split3(dtype, flags)) k *= 3;  // the operands carry [hi|hi|lo] x [hi|lo|hi] per 16-block of K
  CUtensorMap maps[5];
  LaunchPlan plan;
  const int rc = plan_gemm(dtype, a_op, b_op, c, rows, k, m, t, tile_sync, b_ready, b_ready_target, attributes_only,
                           stream, batch, half, maps, &plan);
  if (rc != MM_OK) return rc;
  const int cg = t.cta_group(), bn = t.block_n();
  if (dtype == MM_DTYPE_UINT8) return dispatch_variant<ptx::KIND_I8, unsigned char>(cg, bn, plan);
  return dtype == MM_DTYPE_FLOAT ? dispatch_variant<ptx::KIND_TF32, float>(cg, bn, plan)
                                 : dispatch_variant<ptx::KIND_F16, __half>(cg, bn, plan);
}

}  // namespace

// C[rows x m] = Aop[rows x k] * B on the tensor cores; `b_op` as returned by tcgen05_prepare_b.  `accumulate`:
// C <- C + that product, by the accumulate kernels.  `half`: float's fp16 copies and fits flags, or empty.
int tcgen05_gemm(int dtype, const void *a_op, const void *b_op, void *c, unsigned rows, unsigned k, unsigned m,
                 int flags, const Tuning &t, unsigned int *tile_sync, const unsigned int *b_ready,
                 unsigned b_ready_target, cudaStream_t stream, const GemmBatch &batch, bool accumulate,
                 const HalfOperands &half) {
  return gemm_dispatch(dtype, a_op, b_op, c, rows, k, m, flags, t, tile_sync, b_ready, b_ready_target, false, stream,
                       batch, accumulate, half);
}

int tcgen05_prepare_b_async(int dtype, const BSource &src, void *local_b, void *scratch, size_t scratch_bytes,
                            unsigned k, unsigned m, int flags, const Tuning &t, cudaStream_t stream, cudaStream_t side,
                            cudaEvent_t ev_fork, cudaEvent_t ev_join, PreparedB *out, unsigned copies, void *bt16,
                            unsigned int *fits) {
  *out = PreparedB{};
  const bool in_place = tcgen05_b_in_place(dtype, flags, t);
  const bool parts = src.src != nullptr;
  if (copies != 1) {
    if (parts) return fail(MM_ERR_UNSUPPORTED, "batched calls take B from one array");
    return tcgen05_prepare_b(dtype, src, scratch, k, m, flags, t, &out->b_op, nullptr, nullptr, stream, copies, bt16,
                             fits);
  }
  if (parts && !tcgen05_b_mn(dtype, flags, t)) {
    // K-major copy requested (tuning / 3xTF32): assemble the slices first, then transpose locally
    int rc = gather_b_rows(src, local_b, elem_bytes(dtype), k, m, stream);
    if (rc != MM_OK) return rc;
    BSource whole;
    whole.b = local_b;
    return tcgen05_prepare_b(dtype, whole, scratch, k, m, flags, t, &out->b_op, nullptr, nullptr, stream, 1, bt16, fits);
  }
  void *bt = in_place ? local_b : scratch;
  const Tcgen05Counters cnt = tcgen05_counters(scratch, scratch_bytes);
  const unsigned panels = ceil_div(m, unsigned(t.block_n()));
  // the panel kernel runs (float rounding, or a gather of slices), a second stream exists, the tuning allows it
  const bool overlap = side != nullptr && t.b_overlap() != 0 && tcgen05_b_mn(dtype, flags, t) && (!in_place || parts) &&
                       panels <= B_READY_BYTES / sizeof(unsigned int);
  if (!overlap) return tcgen05_prepare_b(dtype, src, bt, k, m, flags, t, &out->b_op, nullptr, nullptr, stream, 1, bt16, fits);
  MM_CUDA_TRY(cudaMemsetAsync(cnt.b_ready, 0, panels * sizeof(unsigned int), stream));
  MM_CUDA_TRY(cudaEventRecord(ev_fork, stream));
  MM_CUDA_TRY(cudaStreamWaitEvent(side, ev_fork, 0));
  const int rc = tcgen05_prepare_b(dtype, src, bt, k, m, flags, t, &out->b_op, cnt.b_ready, &out->ready_target, side);
  cudaEventRecord(ev_join, side);  // the side stream rejoins whatever happened above
  out->forked = true;
  out->ready = cnt.b_ready;
  return rc;
}

int launch_tcgen05(int dtype, const GemmArgs &g, void *scratch, size_t scratch_bytes) {
  if (dtype != MM_DTYPE_FLOAT && dtype != MM_DTYPE_HALF && dtype != MM_DTYPE_UINT8 && dtype != MM_DTYPE_BFLOAT16) {
    return fail(MM_ERR_UNSUPPORTED, "tcgen05 path handles float, half, bfloat16 and uint8_t only");
  }
  if (g.tuning == nullptr) return fail(MM_ERR_INVALID, "tcgen05 launch without tuning");
  const Tuning &t = *g.tuning;
  if (g.dry_run) {
    // force the lazily loaded kernels in (prep + the GEMM variant this tuning selects) and the driver entry point
    cudaFuncAttributes attr;
    MM_CUDA_TRY(cudaFuncGetAttributes(&attr, round_tf32_kernel<true>));
    MM_CUDA_TRY(cudaFuncGetAttributes(&attr, round_tf32_kernel<false>));
    MM_CUDA_TRY(cudaFuncGetAttributes(&attr, prep_b_panels_kernel<true>));
    MM_CUDA_TRY(cudaFuncGetAttributes(&attr, prep_b_panels_kernel<false>));
    MM_CUDA_TRY(cudaFuncGetAttributes(&attr, transpose_prep_kernel<float, true>));
    MM_CUDA_TRY(cudaFuncGetAttributes(&attr, transpose_prep_kernel<__half, false>));
    MM_CUDA_TRY(cudaFuncGetAttributes(&attr, transpose_prep_kernel<unsigned char, false>));
    if (!get_encode_fn()) return fail(MM_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
    return gemm_dispatch(dtype, nullptr, nullptr, nullptr, g.n, g.k, g.m, g.flags, t, nullptr, nullptr, 0, true, g.stream,
                         g.batch, g.accumulate);
  }
  if (scratch_bytes < tcgen05_scratch_bytes(dtype, g.n, g.k, g.m, g.flags, t, g.batch)) {
    return fail(MM_ERR_INVALID, "tcgen05 scratch too small");
  }
  unsigned char *sp = static_cast<unsigned char *>(scratch);
  void *aprep = sp + tcgen05_bt_bytes(dtype, g.k, g.m, g.flags, t, g.batch.b_copies());
  const Tcgen05Counters cnt = tcgen05_counters(scratch, scratch_bytes);
  BSource src;
  src.b = g.b;
  PreparedB pb;
  const void *a_op = nullptr;
  const HalfScratch hs = tcgen05_half_scratch(scratch, scratch_bytes, dtype, g.n, g.k, g.m, g.flags, t, g.batch);
  if (hs.fits_b) MM_CUDA_TRY(cudaMemsetAsync(hs.fits_b, 1, hs.flag_bytes, g.stream));  // every operand fits until seen
  // one preparation pass per operand for the whole batch; a shared operand is prepared once
  int rc = tcgen05_prepare_b_async(dtype, src, nullptr, scratch, scratch_bytes, g.k, g.m, g.flags, t, g.stream,
                                   g.side_stream, g.ev_fork, g.ev_join, &pb, g.batch.b_copies(), hs.b, hs.fits_b);
  if (rc == MM_OK) {
    rc = tcgen05_prepare_a(dtype, g.a, aprep, g.n, g.k, g.flags, t, &a_op, g.stream, g.batch.a_copies(), hs.a,
                           hs.fits_a);
  }
  if (rc == MM_OK && g.agree != nullptr) rc = (*g.agree)(hs.fits_a, g.stream);
  if (rc == MM_OK && g.ev_prep_done) cudaEventRecord(g.ev_prep_done, g.stream);
  if (rc == MM_OK) {
    rc = tcgen05_gemm(dtype, a_op, pb.b_op, g.c, g.n, g.k, g.m, g.flags, t, cnt.tile_sync, pb.ready, pb.ready_target,
                      g.stream, g.batch, g.accumulate, hs.operands());
  }
  if (pb.forked) cudaStreamWaitEvent(g.stream, g.ev_join, 0);  // join, on the error paths too
  return rc;
}

}  // namespace mm
