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
//     Float A and B are therefore rounded to nearest TF32 (cvt.rna.tf32.f32) into scratch copies first, by
//     prep_float_operands_kernel and complete_tf32_kernel.
//   * A value rounded to TF32 keeps 10 mantissa bits, as many as a half has.  So those passes may write the
//     rounded operands as halves instead, and note, per distinct operand, whether every value is 0 or a normal half
//     (fits_half.h).  A problem whose A and B both fit runs on the f16 wgmma, which multiplies the very same values
//     at twice the TF32 issue rate (gemm_wgmma.cuh); any other problem stays on TF32.
//   * MM_FLAG_TF32X3 splits float A and B into hi / lo parts (split3_*); the tf32_no_round experiment transposes
//     float B unrounded.
//   * half, bfloat16 and uint8_t A are K-major as stored; B is transposed.  bfloat16 moves the same bits as
//     half, so it shares half's transpose kernel.
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

// ---- float on the default datapath: one preparation pass that writes the copy the GEMM will read ---------------
// A problem reads either the TF32 copies of its operands or the fp16 copies, never both (HalfOperands).  So the first
// pass, prep_float_operands_kernel, writes one copy per item: an item is one 64 x 64 tile of a source operand, and it
// is prepared in one of two modes, read once from the fits words at its start and uniform across the block:
//   optimistic   round to TF32, write the fp16 copy only, and clear the copy's fits word when a value does not fit;
//                the item's TF32 copy stays owed (its byte in the pending map stays 1).
//   settled      a fits word that already reads 0 proves that every problem reading this copy runs on TF32 (its own
//                word, or the partner operand's word when this copy is read by one problem only); write the TF32 copy
//                only and clear the item's pending byte.
// Within a call the words only go from nonzero to zero (the memset, these passes, the multi-GPU agreement), so a
// settled item is never needed as fp16.  The second pass, complete_tf32_kernel, runs once the words are final (after
// the multi-GPU agreement): for each copy that some problem reads on TF32 it writes the TF32 copy of every item still
// owed, reading the source again.  Data that fits costs 6 bytes per element (read fp32, write fp16), data found not to
// fit early 8 (read, write TF32).
constexpr int FP_TILE = 64;
constexpr int FP_THREADS = 256;

struct FloatPrepOperand {
  const float *src = nullptr;  // `copies` packed src_rows x src_cols row-major sources
  float *dst = nullptr;        // TF32 copies, K-major: the source itself (flat) or its transpose
  __half *dst16 = nullptr;     // fp16 copies, same layout
  unsigned int *fits = nullptr;            // one word per copy
  const unsigned int *partner = nullptr;   // the other operand's words; null when a copy is read by several problems
  uint32_t partner_stride = 0;             // 1: copy i's problem reads the other operand's copy i; 0: its only copy
  const unsigned int *other = nullptr;     // all of the other operand's words (other_count), for a shared copy
  uint32_t other_count = 0;
  unsigned char *pending = nullptr;        // one byte per item: 1 = its TF32 copy is still owed
  uint32_t src_rows = 0, src_cols = 0, tiles_c = 0, items_per_copy = 0, items = 0;
  bool transpose = false;  // dst = the transpose of src (B, or A stored K x N)
  bool vec = false;        // src rows are whole float4 (src_cols % 4 == 0)
};
struct FloatPrepArgs {
  FloatPrepOperand op[2];
};

struct FloatItemSmem {
  float tile[FP_TILE][FP_TILE + 1];
  int settled;
};

// Whether copy `copy` of `o` is certainly read on TF32 by every problem that reads it, from the words as they are now.
__device__ __forceinline__ bool settled_now(const FloatPrepOperand &o, uint32_t copy) {
  const volatile unsigned int *own = o.fits;
  if (own[copy] == 0u) return true;
  const volatile unsigned int *partner = o.partner;
  return partner != nullptr && partner[copy * o.partner_stride] == 0u;
}

// One item.  COMPLETE (complete_tf32_kernel): the TF32 copy only, nothing else touched.  Otherwise the mode is read
// from the words, and the item's pending byte or the copy's fits word updated at its end.  Ends with a barrier.
template <bool COMPLETE>
__device__ __forceinline__ void float_item(const FloatPrepOperand &o, uint32_t item, FloatItemSmem &sm) {
  const uint32_t t = threadIdx.x;
  const uint32_t copy = item / o.items_per_copy;
  const uint32_t tile_i = item - copy * o.items_per_copy;
  const uint32_t r0 = tile_i / o.tiles_c * FP_TILE, c0 = tile_i % o.tiles_c * FP_TILE;
  const size_t base = size_t(copy) * o.src_rows * o.src_cols;
  const float *src = o.src + base;
  float v[16];
  bool fit = true;
  // loads: flat items as 8-float groups (row q / 8, columns 8 * (q % 8)), transposed items as float4 (row f / 16,
  // columns 4 * (f % 16)); both read whole 256-byte row segments per 16 (8) lanes
  if (!o.transpose) {
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const uint32_t q = t + FP_THREADS * j, r = r0 + q / 8, c = c0 + 8 * (q % 8);
      float4 x = make_float4(0.f, 0.f, 0.f, 0.f), y = x;
      if (r < o.src_rows && c < o.src_cols) {
        const float4 *p = reinterpret_cast<const float4 *>(src + size_t(r) * o.src_cols + c);
        x = p[0];
        y = p[1];
      }
      v[8 * j + 0] = x.x; v[8 * j + 1] = x.y; v[8 * j + 2] = x.z; v[8 * j + 3] = x.w;
      v[8 * j + 4] = y.x; v[8 * j + 5] = y.y; v[8 * j + 6] = y.z; v[8 * j + 7] = y.w;
    }
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t f = t + FP_THREADS * j, r = r0 + f / 16, c = c0 + 4 * (f % 16);
      float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
      if (r < o.src_rows) {
        const float *p = src + size_t(r) * o.src_cols + c;
        if (o.vec) {
          if (c < o.src_cols) x = *reinterpret_cast<const float4 *>(p);
        } else {
          if (c + 0 < o.src_cols) x.x = p[0];
          if (c + 1 < o.src_cols) x.y = p[1];
          if (c + 2 < o.src_cols) x.z = p[2];
          if (c + 3 < o.src_cols) x.w = p[3];
        }
      }
      v[4 * j + 0] = x.x; v[4 * j + 1] = x.y; v[4 * j + 2] = x.z; v[4 * j + 3] = x.w;
    }
  }
#pragma unroll
  for (int e = 0; e < 16; ++e) {
    v[e] = round_tf32(v[e]);
    if (!COMPLETE) fit = fit && tf32_fits_half(__float_as_uint(v[e]));  // padding is 0, which fits
  }
  if (o.transpose) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t f = t + FP_THREADS * j, r = f / 16, c = 4 * (f % 16);
#pragma unroll
      for (int e = 0; e < 4; ++e) sm.tile[r][c + e] = v[4 * j + e];
    }
  }
  if (!COMPLETE && t == 0) sm.settled = settled_now(o, copy);
  __syncthreads();
  const bool settled = COMPLETE || sm.settled;
  float *dst = o.dst + base;
  __half *dst16 = o.dst16 + base;
  const uint32_t ld = o.transpose ? o.src_rows : o.src_cols;  // destination row length (K)
  if (!o.transpose) {
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const uint32_t q = t + FP_THREADS * j, r = r0 + q / 8, c = c0 + 8 * (q % 8);
      if (r >= o.src_rows || c >= o.src_cols) continue;
      const size_t off = size_t(r) * ld + c;
      const float *w = v + 8 * j;
      if (settled) {
        reinterpret_cast<float4 *>(dst + off)[0] = make_float4(w[0], w[1], w[2], w[3]);
        reinterpret_cast<float4 *>(dst + off)[1] = make_float4(w[4], w[5], w[6], w[7]);
      } else {
        *reinterpret_cast<uint4 *>(dst16 + off) =
            make_uint4(half2_bits(w[0], w[1]), half2_bits(w[2], w[3]), half2_bits(w[4], w[5]), half2_bits(w[6], w[7]));
      }
    }
  } else if (settled) {
    // 4 k-values of destination row m per 16-byte store; a warp covers 4 rows x 32 k: conflict-free column reads
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t idx = t + FP_THREADS * j, m = idx % 4 + 4 * (idx / 64), g = idx / 4 % 16;
      if (c0 + m >= o.src_cols || r0 + 4 * g >= o.src_rows) continue;
      float4 x;
      x.x = sm.tile[4 * g + 0][m];
      x.y = sm.tile[4 * g + 1][m];
      x.z = sm.tile[4 * g + 2][m];
      x.w = sm.tile[4 * g + 3][m];
      *reinterpret_cast<float4 *>(dst + size_t(c0 + m) * ld + r0 + 4 * g) = x;
    }
  } else {
    // 8 k-values per 16-byte store of halves; a warp covers 8 rows x 32 k
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const uint32_t idx = t + FP_THREADS * j, m = idx % 8 + 8 * (idx / 64), g = idx / 8 % 8;
      if (c0 + m >= o.src_cols || r0 + 8 * g >= o.src_rows) continue;
      float x[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) x[e] = sm.tile[8 * g + e][m];
      *reinterpret_cast<uint4 *>(dst16 + size_t(c0 + m) * ld + r0 + 8 * g) =
          make_uint4(half2_bits(x[0], x[1]), half2_bits(x[2], x[3]), half2_bits(x[4], x[5]), half2_bits(x[6], x[7]));
    }
  }
  // the barrier also frees sm for the next item
  const int misfit = __syncthreads_or(!settled && !fit);
  if (!COMPLETE && t == 0) {
    if (settled) o.pending[item] = 0;
    else if (misfit) o.fits[copy] = 0u;
  }
}

// First pass: every item of both operands, dealt round-robin to a persistent grid (op[0]'s items first).
__global__ void __launch_bounds__(FP_THREADS)
prep_float_operands_kernel(const FloatPrepArgs args) {
  __shared__ FloatItemSmem sm;
  const uint32_t items0 = args.op[0].items, total = items0 + args.op[1].items;
  for (uint32_t item = blockIdx.x; item < total; item += gridDim.x) {
    if (item < items0) float_item<false>(args.op[0], item, sm);
    else float_item<false>(args.op[1], item - items0, sm);
  }
}

// Whether some problem reading copy `copy` of `o` runs on TF32, from the final words.  `any_other_zero`: one of the
// other operand's words is 0 (what decides for a copy that several problems read).
__device__ __forceinline__ bool read_on_tf32(const FloatPrepOperand &o, uint32_t copy, bool any_other_zero) {
  if (o.fits[copy] == 0u) return true;
  return o.partner != nullptr ? o.partner[copy * o.partner_stride] == 0u : any_other_zero;
}

// Second pass: the TF32 copy of every item still owed whose copy some problem reads on TF32.  Each block gathers up
// to 256 of its items per round with one load per thread, so that a call that owes nothing costs one round.
__global__ void __launch_bounds__(FP_THREADS)
complete_tf32_kernel(const FloatPrepArgs args) {
  __shared__ FloatItemSmem sm;
  __shared__ uint32_t owed[FP_THREADS];
  __shared__ uint32_t owed_count;
  const uint32_t t = threadIdx.x;
  // any_zero(o): one of the other operand's words is 0; only a copy that several problems read asks
  auto any_zero = [t](const FloatPrepOperand &o) {
    bool z = false;
    if (o.items != 0 && o.partner == nullptr) {
      for (uint32_t w = t; w < o.other_count; w += FP_THREADS) z = z || o.other[w] == 0u;
    }
    return __syncthreads_or(z) != 0;
  };
  const bool zero0 = any_zero(args.op[0]), zero1 = any_zero(args.op[1]);
  const uint32_t items0 = args.op[0].items, total = items0 + args.op[1].items;
  if (t == 0) owed_count = 0;
  __syncthreads();
  for (size_t first = blockIdx.x; first < total; first += size_t(FP_THREADS) * gridDim.x) {
    const size_t slot = first + size_t(t) * gridDim.x;
    if (slot < total) {
      const uint32_t item = uint32_t(slot);
      const bool second = item >= items0;
      const FloatPrepOperand &o = second ? args.op[1] : args.op[0];
      const uint32_t local = second ? item - items0 : item;
      if (read_on_tf32(o, local / o.items_per_copy, second ? zero1 : zero0) && o.pending[local] != 0) {
        owed[atomicAdd(&owed_count, 1u)] = item;
      }
    }
    __syncthreads();
    const uint32_t count = owed_count;
    for (uint32_t j = 0; j < count; ++j) {
      const uint32_t it = owed[j];
      if (it < items0) float_item<true>(args.op[0], it, sm);
      else float_item<true>(args.op[1], it - items0, sm);
    }
    __syncthreads();
    if (t == 0) owed_count = 0;
    __syncthreads();
  }
}

// Row-sliced B (row-major K x M, 16-byte vectors) -> dst (same layout): k-row r is read from parts[r / part_rows], a
// full-size K x M array on a (peer) GPU of which only that slice of rows is valid; rows whose source IS the
// destination are skipped.  A work item is GATHER_ROWS k-rows of GATHER_VECS vectors (1 KiB) per row, 8 loads in
// flight per thread; items are numbered column-block-major and dealt round-robin to the CTAs of a persistent grid.
constexpr int GATHER_THREADS = 512;
constexpr int GATHER_WARPS = GATHER_THREADS / 32;
constexpr int GATHER_ROWS = 64;
constexpr int GATHER_VECS = 64;
constexpr int GATHER_ROW_SLOTS = GATHER_ROWS / GATHER_WARPS;  // rows per warp per item (4)

__global__ void __launch_bounds__(GATHER_THREADS)
gather_rows_kernel(const uint4 *const *__restrict__ parts, uint32_t part_rows, uint4 *__restrict__ dst, uint32_t k,
                   uint32_t row_v) {
  const uint32_t warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const uint32_t col_blocks = (row_v + GATHER_VECS - 1) / GATHER_VECS;
  const uint32_t items_per_col_block = (k + GATHER_ROWS - 1) / GATHER_ROWS;
  const uint32_t items = col_blocks * items_per_col_block;
  for (uint32_t item = blockIdx.x; item < items; item += gridDim.x) {
    const uint32_t col_block = item / items_per_col_block;
    const uint32_t r0 = (item - col_block * items_per_col_block) * GATHER_ROWS;
    const uint32_t v0 = col_block * GATHER_VECS;
    const uint32_t w = min(uint32_t(GATHER_VECS), row_v - v0);
    uint4 buf[GATHER_ROW_SLOTS][2];
    bool live[GATHER_ROW_SLOTS][2];
#pragma unroll
    for (int u = 0; u < GATHER_ROW_SLOTS; ++u) {
      const uint32_t r = r0 + warp + u * GATHER_WARPS;
      const uint4 *src = r < k ? parts[r / part_rows] : nullptr;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t c = lane + 32 * h;
        const size_t off = size_t(r) * row_v + v0 + c;
        live[u][h] = (r < k) && (c < w) && (src != dst);
        if (live[u][h]) buf[u][h] = src[off];
      }
    }
#pragma unroll
    for (int u = 0; u < GATHER_ROW_SLOTS; ++u) {
      const uint32_t r = r0 + warp + u * GATHER_WARPS;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t c = lane + 32 * h;
        if (live[u][h]) dst[size_t(r) * row_v + v0 + c] = buf[u][h];
      }
    }
  }
}

// dst[c][r] = src[r][c] for src of shape src_rows x src_cols (row-major): 64 x 64 tiles through
// shared memory so that both the reads and the writes are row-contiguous.  blockIdx.z = problem of a
// batch: packed sources, packed destinations.
template <typename T>
__global__ void __launch_bounds__(256)
transpose_prep_kernel(const T *__restrict__ src, T *__restrict__ dst, uint32_t src_rows, uint32_t src_cols) {
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
    if (r < src_rows && c < src_cols) tile[i][x] = src[size_t(r) * src_cols + c];
  }
  __syncthreads();
#pragma unroll 4
  for (int i = y; i < TILE; i += 4) {
    const uint32_t c = c0 + i, r = r0 + x;  // dst row = src col
    if (c < src_cols && r < src_rows) dst[size_t(c) * src_rows + r] = tile[x][i];
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

template <typename T>
void launch_transpose(const void *src, void *dst, uint32_t src_rows, uint32_t src_cols, cudaStream_t stream,
                      unsigned copies) {
  dim3 grid((src_cols + 63) / 64, (src_rows + 63) / 64, copies);
  transpose_prep_kernel<T><<<grid, 256, 0, stream>>>(static_cast<const T *>(src), static_cast<T *>(dst), src_rows,
                                                     src_cols);
}

bool split3(int dtype, int flags) { return dtype == MM_DTYPE_FLOAT && (flags & MM_FLAG_TF32X3); }

}  // namespace

// Tail of the scratch: the soft wave-barrier counter of the GEMM, 256 B
constexpr size_t TAIL_BYTES = 256;
static_assert(TAIL_BYTES == kTcgen05TailBytes, "common.cuh and gemm_tcgen05.cu disagree on the scratch tail");

unsigned int *tcgen05_tile_sync(void *scratch, size_t scratch_bytes) {
  return reinterpret_cast<unsigned int *>(static_cast<unsigned char *>(scratch) + scratch_bytes - TAIL_BYTES);
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
// 64 x 64 items of one copy of a rows x cols operand (either orientation: the count is the same)
uint32_t float_items(unsigned rows, unsigned cols) { return ceil_div(rows, FP_TILE) * ceil_div(cols, FP_TILE); }
// [fits words of B][fits words of A][pending map of B][pending map of A]
size_t fits_bytes(unsigned n, unsigned k, unsigned m, const GemmBatch &batch) {
  return align_up(size_t(batch.a_copies() + batch.b_copies()) * sizeof(unsigned int) +
                      size_t(batch.b_copies()) * float_items(k, m) + size_t(batch.a_copies()) * float_items(n, k),
                  1024);
}

size_t tcgen05_bt_bytes(int dtype, unsigned k, unsigned m, int flags, const Tuning &t, unsigned b_copies) {
  const size_t fp16 = half_copies(dtype, flags, t) ? align_up(size_t(b_copies) * m * k * 2, 1024) : 0;
  return b_copy_bytes(dtype, k, m, flags, b_copies) + fp16;  // [B copy][B fp16]
}

size_t tcgen05_scratch_bytes(int dtype, unsigned n, unsigned k, unsigned m, int flags, const Tuning &t,
                             const GemmBatch &batch) {
  size_t bytes = TAIL_BYTES + tcgen05_bt_bytes(dtype, k, m, flags, t, batch.b_copies());  // counter (tail) + B copies
  bytes += a_copy_bytes(dtype, n, k, flags, batch.a_copies());
  if (half_copies(dtype, flags, t)) bytes += align_up(size_t(batch.a_copies()) * n * k * 2, 1024) + fits_bytes(n, k, m, batch);
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
  h.flag_bytes = fits_bytes(n, k, m, batch);
  h.fits_b = reinterpret_cast<unsigned int *>(sp + scratch_bytes - TAIL_BYTES - h.flag_bytes);
  h.fits_a = h.fits_b + batch.b_copies();
  h.pending_b = reinterpret_cast<unsigned char *>(h.fits_a + batch.a_copies());
  h.pending_a = h.pending_b + size_t(batch.b_copies()) * float_items(k, m);
  return h;
}

int gather_b_rows(const void *const *parts, unsigned part_rows, void *dst, size_t elem_bytes, unsigned k, unsigned m,
                  cudaStream_t stream) {
  const uint32_t row_v = uint32_t(size_t(m) * elem_bytes / 16);
  gather_rows_kernel<<<num_sms() * 2, GATHER_THREADS, 0, stream>>>(reinterpret_cast<const uint4 *const *>(parts),
                                                                   part_rows, static_cast<uint4 *>(dst), k, row_v);
  MM_CUDA_TRY(cudaGetLastError());
  return MM_OK;
}

int tcgen05_prepare_b(int dtype, const void *b, void *bt, unsigned k, unsigned m, int flags, const Tuning &t,
                      const void **b_op, cudaStream_t stream, unsigned copies) {
  *b_op = bt;
  if (split3(dtype, flags)) {
    dim3 grid((m + 63) / 64, (k + 63) / 64, copies);
    split3_transpose_kernel<true><<<grid, 256, 0, stream>>>(static_cast<const float *>(b), static_cast<float *>(bt), k, m);
  } else if (dtype == MM_DTYPE_FLOAT) {
    if (!t.tf32_no_round()) return fail(MM_ERR_INVALID, "float's rounded operands come from tcgen05_prepare_float");
    launch_transpose<float>(b, bt, k, m, stream, copies);
  } else if (dtype == MM_DTYPE_UINT8) {
    launch_transpose<unsigned char>(b, bt, k, m, stream, copies);
  } else {
    launch_transpose<__half>(b, bt, k, m, stream, copies);
  }
  MM_CUDA_TRY(cudaGetLastError());
  return MM_OK;
}

// `rows` rows of A -> the K-major A operand.  Row-major float A is rounded into `aprep`; row-major
// half, bfloat16 and uint8_t A are used in place; A stored K x N (`transposed`, leading dimension = rows, only whole
// matrices) is transposed into `aprep`.  *a_op receives the operand pointer.  `copies` packed problems:
// the row-wise passes run over copies * rows rows, the transposes take the problem from blockIdx.z.
int tcgen05_prepare_a(int dtype, const void *a, void *aprep, unsigned rows, unsigned k, int flags, const Tuning &t,
                      const void **a_op, cudaStream_t stream, unsigned copies) {
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
    if (!t.tf32_no_round()) return fail(MM_ERR_INVALID, "float's rounded operands come from tcgen05_prepare_float");
    if (transposed) {
      launch_transpose<float>(a, aprep, k, rows, stream, copies);  // A stored K x N -> N x K
      *a_op = aprep;
    }
  } else if (transposed) {
    if (dtype == MM_DTYPE_UINT8) launch_transpose<unsigned char>(a, aprep, k, rows, stream, copies);
    else launch_transpose<__half>(a, aprep, k, rows, stream, copies);
    *a_op = aprep;
  }
  MM_CUDA_TRY(cudaGetLastError());
  return MM_OK;
}

namespace {
FloatPrepOperand float_operand(const void *src, float *dst, __half *dst16, unsigned src_rows, unsigned src_cols,
                               unsigned copies, bool transpose, unsigned int *fits, unsigned char *pending) {
  FloatPrepOperand o;
  o.src = static_cast<const float *>(src);
  o.dst = dst;
  o.dst16 = dst16;
  o.fits = fits;
  o.pending = pending;
  o.src_rows = src_rows;
  o.src_cols = src_cols;
  o.tiles_c = ceil_div(src_cols, FP_TILE);
  o.items_per_copy = float_items(src_rows, src_cols);
  o.items = copies * o.items_per_copy;
  o.transpose = transpose;
  o.vec = src_cols % 4 == 0;
  return o;
}

// A persistent grid: as many blocks as are resident at once, at most one per item.
int float_prep_grid(const void *kernel, uint32_t items) {
  MM_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                                   cudaSharedmemCarveoutMaxShared));
  int per_sm = 0;
  MM_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, FP_THREADS, 0));
  return int(std::max<uint32_t>(1u, std::min<uint32_t>(items, uint32_t(std::max(per_sm, 1) * num_sms()))));
}
}  // namespace

int tcgen05_prepare_float(bool complete, const void *a, unsigned row0, unsigned rows, const void *b, unsigned n,
                          unsigned k, unsigned m, int flags, const Tuning &t, const GemmBatch &batch, void *scratch,
                          size_t scratch_bytes, cudaStream_t stream) {
  const HalfScratch hs = tcgen05_half_scratch(scratch, scratch_bytes, MM_DTYPE_FLOAT, n, k, m, flags, t, batch);
  if (hs.fits_a == nullptr) return fail(MM_ERR_INVALID, "tcgen05_prepare_float: float on the default datapath only");
  if (row0 % FP_TILE != 0) return fail(MM_ERR_INVALID, "tcgen05_prepare_float: A's first row must be a multiple of 64");
  unsigned char *sp = static_cast<unsigned char *>(scratch);
  // a copy that several problems read settles on its own word only
  const bool shared_a = batch.count > 1 && batch.shared_a, shared_b = batch.count > 1 && batch.shared_b;
  FloatPrepArgs args;
  if (b != nullptr) {
    FloatPrepOperand &o = args.op[0];
    o = float_operand(b, reinterpret_cast<float *>(sp), static_cast<__half *>(hs.b), k, m, batch.b_copies(), true,
                      hs.fits_b, hs.pending_b);
    o.partner = shared_b ? nullptr : hs.fits_a;
    o.partner_stride = shared_a ? 0 : 1;
    o.other = hs.fits_a;
    o.other_count = batch.a_copies();
  }
  if (a != nullptr) {
    const bool transposed = (flags & MM_FLAG_TRANSPOSED_A) != 0;
    if (transposed && (row0 != 0 || rows != n)) return fail(MM_ERR_INVALID, "A stored K x N is prepared whole");
    const size_t first = size_t(row0) * k;  // row0's element in the N x K copies; its items start at row0 / 64
    float *aprep = reinterpret_cast<float *>(sp + tcgen05_bt_bytes(MM_DTYPE_FLOAT, k, m, flags, t, batch.b_copies()));
    FloatPrepOperand &o = args.op[1];
    o = float_operand(a, aprep + first, static_cast<__half *>(hs.a) + first, transposed ? k : rows,
                      transposed ? rows : k, batch.a_copies(), transposed, hs.fits_a,
                      hs.pending_a + size_t(row0 / FP_TILE) * ceil_div(k, FP_TILE));
    o.partner = shared_a ? nullptr : hs.fits_b;
    o.partner_stride = shared_b ? 0 : 1;
    o.other = hs.fits_b;
    o.other_count = batch.b_copies();
  }
  const uint32_t items = args.op[0].items + args.op[1].items;
  if (complete) {
    const int grid = float_prep_grid(reinterpret_cast<const void *>(complete_tf32_kernel), items);
    complete_tf32_kernel<<<grid, FP_THREADS, 0, stream>>>(args);
  } else {
    const int grid = float_prep_grid(reinterpret_cast<const void *>(prep_float_operands_kernel), items);
    prep_float_operands_kernel<<<grid, FP_THREADS, 0, stream>>>(args);
  }
  MM_CUDA_TRY(cudaGetLastError());
  return MM_OK;
}

namespace {
int gemm_dispatch(int dtype, const void *a_op, const void *b_op, void *c, unsigned rows, unsigned k, unsigned m,
                  int flags, const Tuning &t, unsigned int *tile_sync, bool attributes_only, cudaStream_t stream,
                  const GemmBatch &batch, bool accumulate = false, const HalfOperands &half = HalfOperands{}) {
  if (accumulate) {
    if (split3(dtype, flags)) k *= 3;
    return wgmma_accumulate_gemm(dtype, a_op, b_op, c, rows, k, m, t, tile_sync, attributes_only, stream, batch, half);
  }
  if (dtype == MM_DTYPE_BFLOAT16) {
    return wgmma_bf16_gemm(a_op, b_op, c, rows, k, m, t, tile_sync, attributes_only, stream, batch);
  }
  if (split3(dtype, flags)) k *= 3;  // the operands carry [hi|hi|lo] x [hi|lo|hi] per 16-block of K
  CUtensorMap maps[5];
  LaunchPlan plan;
  const int rc = plan_gemm(dtype, a_op, b_op, c, rows, k, m, t, tile_sync, attributes_only, stream, batch, half, maps,
                           &plan);
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
                 int flags, const Tuning &t, unsigned int *tile_sync, cudaStream_t stream, const GemmBatch &batch,
                 bool accumulate, const HalfOperands &half) {
  return gemm_dispatch(dtype, a_op, b_op, c, rows, k, m, flags, t, tile_sync, false, stream, batch, accumulate, half);
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
    MM_CUDA_TRY(cudaFuncGetAttributes(&attr, gather_rows_kernel));
    MM_CUDA_TRY(cudaFuncGetAttributes(&attr, prep_float_operands_kernel));
    MM_CUDA_TRY(cudaFuncGetAttributes(&attr, complete_tf32_kernel));
    MM_CUDA_TRY(cudaFuncGetAttributes(&attr, transpose_prep_kernel<__half>));
    MM_CUDA_TRY(cudaFuncGetAttributes(&attr, transpose_prep_kernel<unsigned char>));
    if (!get_encode_fn()) return fail(MM_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
    return gemm_dispatch(dtype, nullptr, nullptr, nullptr, g.n, g.k, g.m, g.flags, t, nullptr, true, g.stream, g.batch,
                         g.accumulate);
  }
  if (scratch_bytes < tcgen05_scratch_bytes(dtype, g.n, g.k, g.m, g.flags, t, g.batch)) {
    return fail(MM_ERR_INVALID, "tcgen05 scratch too small");
  }
  unsigned char *sp = static_cast<unsigned char *>(scratch);
  void *aprep = sp + tcgen05_bt_bytes(dtype, g.k, g.m, g.flags, t, g.batch.b_copies());
  const void *a_op = nullptr, *b_op = nullptr;
  const HalfScratch hs = tcgen05_half_scratch(scratch, scratch_bytes, dtype, g.n, g.k, g.m, g.flags, t, g.batch);
  // the whole batch is prepared at once; a shared operand is prepared once
  int rc = MM_OK;
  if (hs.fits_b) {
    // every operand fits and every item's TF32 copy is owed until seen; then one pass over A and B
    MM_CUDA_TRY(cudaMemsetAsync(hs.fits_b, 1, hs.flag_bytes, g.stream));
    b_op = scratch;
    a_op = aprep;
    rc = tcgen05_prepare_float(false, g.a, 0, g.n, g.b, g.n, g.k, g.m, g.flags, t, g.batch, scratch, scratch_bytes,
                               g.stream);
  } else {
    rc = tcgen05_prepare_b(dtype, g.b, scratch, g.k, g.m, g.flags, t, &b_op, g.stream, g.batch.b_copies());
    if (rc == MM_OK) rc = tcgen05_prepare_a(dtype, g.a, aprep, g.n, g.k, g.flags, t, &a_op, g.stream, g.batch.a_copies());
  }
  if (rc == MM_OK && g.agree != nullptr) rc = (*g.agree)(hs.fits_a, g.stream);
  if (rc == MM_OK && hs.fits_b) {  // the words are final: the TF32 copies still owed
    rc = tcgen05_prepare_float(true, g.a, 0, g.n, g.b, g.n, g.k, g.m, g.flags, t, g.batch, scratch, scratch_bytes,
                               g.stream);
  }
  if (rc == MM_OK && g.ev_prep_done) cudaEventRecord(g.ev_prep_done, g.stream);
  if (rc == MM_OK) {
    rc = tcgen05_gemm(dtype, a_op, b_op, g.c, g.n, g.k, g.m, g.flags, t, tcgen05_tile_sync(scratch, scratch_bytes),
                      g.stream, g.batch, g.accumulate, hs.operands());
  }
  return rc;
}

}  // namespace mm
