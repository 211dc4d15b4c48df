// Tensor-core path of the hot path for the dense (Multiply, Add) contraction on float, half and uint8_t:
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
//   * half and uint8_t A are K-major as stored; B is transposed.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "ptx_sm90.cuh"
#include "tma_host.cuh"

namespace mm {
namespace {

constexpr int BLOCK_M = 128;          // C rows per CTA (two consumer warpgroups of 64 rows)
constexpr int BLOCK_K_BYTES = 128;    // one 128-byte swizzle atom of K per stage
constexpr int WGMMA_K_BYTES = 32;     // K extent of one wgmma
constexpr int NUM_THREADS = 384;      // producer warpgroup + 2 consumer warpgroups
constexpr int CONSUMER_WARPS = 8;
constexpr int EPI_ROWS = 16;          // one staged C block per consumer warp: 16 rows x 32 columns
constexpr int EPI_BUF_BYTES = 2048;
constexpr int EPI_BYTES = CONSUMER_WARPS * EPI_BUF_BYTES;
constexpr int BAR_BYTES = 256;
constexpr int MAX_DYN_SMEM = 232448;  // 227 KiB per CTA on sm_90a

// Per-variant geometry.  CG = 1: one CTA computes a 128 x BN tile.  CG = 2: a cluster of two CTAs
// computes 256 x BN; every CTA holds the whole B tile per stage but fetches only its half of it.
template <int CG, int BN>
struct Geo {
  static constexpr int LOAD_N = BN / CG;                            // B rows (columns of C) fetched per CTA
  static constexpr int A_STAGE_BYTES = BLOCK_M * BLOCK_K_BYTES;     // 16 KiB
  static constexpr int B_STAGE_BYTES = BN * BLOCK_K_BYTES;          // 16 | 32 KiB
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int FIT = (MAX_DYN_SMEM - 1024 - BAR_BYTES - EPI_BYTES) / STAGE_BYTES;
  static constexpr int MAX_STAGES = FIT < 8 ? FIT : 8;              // 4 (BN 256)  6 (BN 128)
  static constexpr int TILE_ROWS = BLOCK_M * CG;                    // C rows per CTA group
  static constexpr size_t smem_bytes(int stages) {
    return size_t(stages) * STAGE_BYTES + EPI_BYTES + 1024 /*align*/ + BAR_BYTES;
  }
};

struct TileCoord {
  uint32_t r, c;
  uint32_t prob;  // problem of a batched call
};

// Grouped rasterisation: RASTER_GROUP row-tiles sweep all column-tiles together so that the
// concurrently running tiles share A row-panels and B column-panels through L2.  Column tiles are
// visited in ascending order within a group.  In a batch the problem is the outermost index: the
// tiles of problem i are tiles [i * tiles_r * tiles_c, (i + 1) * tiles_r * tiles_c), rasterised as above.
__device__ __forceinline__ TileCoord tile_coord(uint32_t t, uint32_t tiles_r, uint32_t tiles_c,
                                                uint32_t raster_group) {
  const uint32_t prob = t / (tiles_r * tiles_c);
  t -= prob * (tiles_r * tiles_c);
  const uint32_t per_group = raster_group * tiles_c;
  const uint32_t g = t / per_group;
  const uint32_t first = g * raster_group;
  const uint32_t gsize = min(raster_group, tiles_r - first);
  const uint32_t in = t - g * per_group;
  return TileCoord{first + in % gsize, in / gsize, prob};
}

// ---- epilogue ------------------------------------------------------------------------------------
// Two adjacent accumulator values (columns c, c + 1 of one row) as the bytes of C.
template <typename TOut>
struct Pair;
template <>
struct Pair<float> {
  using T = uint2;
  __device__ __forceinline__ static uint2 make(uint32_t a, uint32_t b) { return make_uint2(a, b); }
};
template <>
struct Pair<__half> {
  using T = uint32_t;
  __device__ __forceinline__ static uint32_t make(uint32_t a, uint32_t b) {
    __half2 h = __floats2half2_rn(__uint_as_float(a), __uint_as_float(b));
    return *reinterpret_cast<uint32_t *>(&h);
  }
};
// uint8_t: the accumulator is the exact 32-bit sum; its low byte is the reference's result (arithmetic modulo 256).
template <>
struct Pair<unsigned char> {
  using T = unsigned short;
  __device__ __forceinline__ static unsigned short make(uint32_t a, uint32_t b) {
    return static_cast<unsigned short>((a & 0xFFu) | ((b & 0xFFu) << 8));
  }
};

__device__ __forceinline__ void st_shared_pair(uint32_t addr, uint2 v) {
  asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr), "r"(v.x), "r"(v.y) : "memory");
}
__device__ __forceinline__ void st_shared_pair(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void st_shared_pair(uint32_t addr, unsigned short v) {
  asm volatile("st.shared.b16 [%0], %1;" ::"r"(addr), "h"(v) : "memory");
}

__device__ __forceinline__ float round_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ unsigned int ld_acquire_gpu(const unsigned int *p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// Run-time launch parameters of the GEMM kernel (one struct so that the instantiations share a
// signature).
struct GemmParams {
  uint32_t rows, cols, k_bytes;
  uint32_t num_stages;       // ring depth actually used (<= Geo::MAX_STAGES, what the smem allocation holds)
  uint32_t raster_group;     // row tiles per rasterisation group
  uint32_t tma_store;        // 1: staged TMA-store epilogue, 0: direct stores
  uint32_t b_ready_target;   // see b_ready
  // Batch: `batch` problems of rows x cols.  A and B are read through 2-D maps with the problems
  // stacked along the row dimension: problem i starts at row i * a_prob_rows of A and
  // i * b_prob_rows of B (0 = every problem reads the same operand).  C is a 3-D map {cols, rows, batch}.
  uint32_t batch, a_prob_rows, b_prob_rows;
  uint64_t l2_policy;
  unsigned int *tile_sync;        // soft wave-barrier counter or null
  const unsigned int *b_ready;    // per column tile: preparation items finished, or null (B complete)
};

// C[rows x cols] = A'[rows x k] * B'^T ; A' (rows x k) and B' (cols x k) K-major.  CG == 2 must be
// launched with cluster dimension (2, 1, 1).
template <int KIND, typename TOut, int CG, int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                  const __grid_constant__ CUtensorMap tmap_c, TOut *__restrict__ C, const GemmParams p) {
  using G = Geo<CG, BN>;
  constexpr int ELEM_BYTES = (KIND == ptx::KIND_TF32) ? 4 : (KIND == ptx::KIND_I8 ? 1 : 2);
  constexpr int BLOCK_K_ELEMS = BLOCK_K_BYTES / ELEM_BYTES;
  const int STAGES = int(p.num_stages);
  const uint32_t rows = p.rows, cols = p.cols;
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  // 128B-swizzled tiles must start on a 1024-byte boundary (same offset in both CTAs of a cluster).
  const uint32_t smem_base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t smem_a0 = smem_base;
  const uint32_t smem_b0 = smem_base + STAGES * G::A_STAGE_BYTES;
  const uint32_t epi0 = smem_base + STAGES * G::STAGE_BYTES;
  const uint32_t bar_base = epi0 + EPI_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };

  const uint32_t warp = threadIdx.x / 32;
  const uint32_t lane = threadIdx.x % 32;
  const uint32_t cta_rank = (CG == 2) ? cluster_ctarank() : 0u;
  const uint32_t group_id = blockIdx.x / CG;
  const uint32_t num_groups = gridDim.x / CG;

  const uint32_t tiles_r = (rows + G::TILE_ROWS - 1) / G::TILE_ROWS;
  const uint32_t tiles_c = (cols + BN - 1) / BN;
  const uint32_t num_tiles = p.batch * tiles_r * tiles_c;
  const uint32_t num_kb = (p.k_bytes + BLOCK_K_BYTES - 1) / BLOCK_K_BYTES;

  if (threadIdx.x == 0) {
    ptx::prefetch_tensormap(&tmap_a);
    ptx::prefetch_tensormap(&tmap_b);
    if (p.tma_store) ptx::prefetch_tensormap(&tmap_c);
    for (int s = 0; s < STAGES; ++s) {
      // full: the own producer's arrive.expect_tx (bytes of A, both halves of B -- the peer's half
      // arrives by its multicast).  empty: one arrival per consumer warp of EVERY CTA of the cluster,
      // because the stage is written by the producers of all of them.
      ptx::mbar_init(full_bar(s), 1);
      ptx::mbar_init(empty_bar(s), CONSUMER_WARPS * CG);
    }
    ptx::fence_mbar_init();
  }
  if (CG == 2) cluster_sync_all(); else __syncthreads();  // the peer's barriers exist before any multicast

  if (warp < 4) {
    // ================= TMA producer (one thread per CTA) =================
    ptx::setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      uint32_t stage = 0, phase = 0;
      uint32_t tile_iter = 0;
      int32_t ready_panel = -1;
      for (uint32_t t = group_id; t < num_tiles; t += num_groups, ++tile_iter) {
        // Soft wave barrier: do not start fetching tile #j before every CTA group has finished
        // fetching its tile #(j-1), so that co-running tiles keep sharing their A / B panels in L2.
        // Purely a performance hint: the wait is bounded, correctness never depends on it.
        if (p.tile_sync != nullptr && tile_iter > 0) {
          const uint32_t target = min(tile_iter * num_groups, num_tiles);
          const long long t0 = clock64();
          while (*reinterpret_cast<volatile unsigned int *>(p.tile_sync) < target) {
            if (clock64() - t0 > 100000) break;  // ~50 us: give up, stay correct
          }
        }
        const TileCoord tc = tile_coord(t, tiles_r, tiles_c, p.raster_group);
        // Rows past the end of a problem belong to the next one: they only feed rows / columns of C
        // that are never stored.  K is the inner dimension, so the K tail is zero-filled per row.
        const int32_t a_row = tc.prob * p.a_prob_rows + tc.r * G::TILE_ROWS + cta_rank * BLOCK_M;
        const int32_t b_row = tc.prob * p.b_prob_rows + tc.c * BN + cta_rank * G::LOAD_N;
        if (p.b_ready != nullptr && int32_t(tc.c) != ready_panel) {
          // B's preparation kernel was ENQUEUED before this kernel and needs no resource this kernel
          // holds, so it always makes progress; the bound only turns an impossible wait into a trap.
          const unsigned int *flag = p.b_ready + tc.c;
          const long long t0 = clock64();
          while (ld_acquire_gpu(flag) < p.b_ready_target) {
            if (clock64() - t0 > (1ll << 34)) __trap();
          }
          asm volatile("fence.proxy.async.global;" ::: "memory");  // generic-proxy writes -> TMA reads
          ready_panel = int32_t(tc.c);
        }
        for (uint32_t kb = 0; kb < num_kb; ++kb) {
          ptx::mbar_wait(empty_bar(stage), phase ^ 1);
          const uint32_t sa = smem_a0 + stage * G::A_STAGE_BYTES;
          const uint32_t sb = smem_b0 + stage * G::B_STAGE_BYTES + cta_rank * G::LOAD_N * BLOCK_K_BYTES;
          const int32_t k0 = kb * BLOCK_K_ELEMS;
          ptx::mbar_arrive_expect_tx(full_bar(stage), G::STAGE_BYTES);
          ptx::tma_load_2d(sa, &tmap_a, full_bar(stage), k0, a_row, p.l2_policy);
          if (CG == 1) {
            ptx::tma_load_2d(sb, &tmap_b, full_bar(stage), k0, b_row, p.l2_policy);
          } else {
            ptx::tma_load_2d_multicast(sb, &tmap_b, full_bar(stage), k0, b_row, 0x3, p.l2_policy);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        if (p.tile_sync != nullptr && cta_rank == 0) atomicAdd(p.tile_sync, 1u);  // this group fetched its tile
      }
    }
  } else {
    // ================= consumers (warpgroups 1, 2) =================
    ptx::setmaxnreg_inc<232>();
    const uint32_t wg = warp / 4 - 1;                  // 64-row half of the tile
    const uint32_t cwarp = warp - 4;                   // 0..7: 16-row slab of the tile
    const uint32_t buf = epi0 + cwarp * EPI_BUF_BYTES;
    const uint32_t peer = cta_rank ^ 1u;
    uint32_t stage = 0, phase = 0;
    uint32_t acc[BN / 2];
    for (uint32_t t = group_id; t < num_tiles; t += num_groups) {
      const TileCoord tc = tile_coord(t, tiles_r, tiles_c, p.raster_group);
      uint32_t prev = 0;
      for (uint32_t kb = 0; kb < num_kb; ++kb) {
        ptx::mbar_wait(full_bar(stage), phase);
        const uint64_t adesc = ptx::make_smem_desc_k_sw128(smem_a0 + stage * G::A_STAGE_BYTES + wg * 64 * BLOCK_K_BYTES);
        const uint64_t bdesc = ptx::make_smem_desc_k_sw128(smem_b0 + stage * G::B_STAGE_BYTES);
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K_BYTES / WGMMA_K_BYTES; ++k) {
          ptx::wgmma<KIND, BN>(acc, adesc + uint64_t(k * (WGMMA_K_BYTES >> 4)), bdesc + uint64_t(k * (WGMMA_K_BYTES >> 4)),
                               (kb | uint32_t(k)) != 0u ? 1u : 0u);
        }
        ptx::wgmma_commit();
        // keep one group in flight: the previous k-block's group has retired, its stage is free
        ptx::wgmma_wait<1>();
        if (kb > 0 && lane == 0) {
          ptx::mbar_arrive(empty_bar(prev));
          if (CG == 2) ptx::mbar_arrive_cluster(empty_bar(prev), peer);
        }
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      ptx::wgmma_wait<0>();
      if (lane == 0) {
        ptx::mbar_arrive(empty_bar(prev));
        if (CG == 2) ptx::mbar_arrive_cluster(empty_bar(prev), peer);
      }

      // ---- epilogue: this warp's 16 rows x BN columns ----
      using P = Pair<TOut>;
      const uint32_t row0 = tc.r * G::TILE_ROWS + cta_rank * BLOCK_M + cwarp * EPI_ROWS;
      const uint32_t r_in = lane / 4, c_in = 2 * (lane % 4);
      if (p.tma_store) {
        // Block of 16 rows x 32 columns, rows of 32 * sizeof(TOut) bytes in the swizzle of that width
        // (128 / 64 / 32 B: 16-byte chunk index XOR address bits 7.. of the row), which the C tensor map expects.
        constexpr uint32_t PITCH = 32 * sizeof(TOut);
        constexpr uint32_t SW_MASK = PITCH / 16 - 1;
#pragma unroll
        for (int chunk = 0; chunk < BN / 32; ++chunk) {
          const uint32_t col = tc.c * BN + chunk * 32;
          if (row0 < rows && col < cols) {                        // warp-uniform
            if (lane == 0) ptx::tma_store_wait_read<0>();         // the previous block has left the buffer
            __syncwarp();
#pragma unroll
            for (int j = 0; j < 4; ++j) {
#pragma unroll
              for (int i = 0; i < 2; ++i) {
                const uint32_t a = buf + (r_in + 8 * i) * PITCH + (8 * j + c_in) * sizeof(TOut);
                const int reg = 4 * (4 * chunk + j) + 2 * i;
                st_shared_pair(a ^ (((a >> 7) & SW_MASK) << 4), P::make(acc[reg], acc[reg + 1]));
              }
            }
            ptx::fence_proxy_async_smem();                        // generic-proxy smem writes -> TMA read
            __syncwarp();
            if (lane == 0) {
              // clipped to rows x cols of this problem by the map
              ptx::tma_store_3d(&tmap_c, buf, int32_t(col), int32_t(row0), int32_t(tc.prob));
              ptx::tma_store_commit();
            }
          }
        }
      } else {
        TOut *Cp = C + size_t(tc.prob) * rows * cols;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const uint32_t row = row0 + r_in + 8 * i;
          if (row >= rows) continue;
          typename P::T *crow = reinterpret_cast<typename P::T *>(Cp + size_t(row) * cols);
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const uint32_t col = tc.c * BN + 8 * j + c_in;
            if (col < cols) crow[col / 2] = P::make(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]);
          }
        }
      }
    }
    if (p.tma_store && lane == 0) ptx::tma_store_wait_all<0>();  // stores complete before the CTA's smem goes away
  }

  // no CTA of a cluster leaves while its peer may still multicast into it or arrive on its barriers
  if (CG == 2) cluster_sync_all();
}

// ---- operand preparation ------------------------------------------------------------------------

// dst[i] = rna_tf32(src[i]); count is a multiple of 4 (K % 16 == 0).
__global__ void __launch_bounds__(256)
round_tf32_kernel(const float4 *__restrict__ src, float4 *__restrict__ dst, size_t count4) {
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < count4; i += stride) {
    float4 v = src[i];
    v.x = round_tf32(v.x);
    v.y = round_tf32(v.y);
    v.z = round_tf32(v.z);
    v.w = round_tf32(v.w);
    dst[i] = v;
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
// batch: packed sources, packed destinations.
template <typename T, bool ROUND>
__global__ void __launch_bounds__(256)
transpose_prep_kernel(const T *__restrict__ src, T *__restrict__ dst, uint32_t src_rows,
                      uint32_t src_cols) {
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
constexpr int SPLIT_BLOCK = 16;  // K % 16 == 0 by the reference's shape rule for float

__device__ __forceinline__ void split_tf32(float x, float &hi, float &lo) {
  hi = round_tf32(x);
  lo = round_tf32(x - hi);
}

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
    row[SPLIT_BLOCK / 4] = hi;
    row[2 * SPLIT_BLOCK / 4] = lo;
  }
}

// src (src_rows = K) x (src_cols) row-major -> dst[c][3K] with per-16-block [a | b | c] where
// B_ORDER selects (hi, lo, hi) for the B operand and (hi, hi, lo) for a transposed A.  blockIdx.z =
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
      out[SPLIT_BLOCK] = B_ORDER ? lo : hi;
      out[2 * SPLIT_BLOCK] = B_ORDER ? hi : lo;
    }
  }
}

// ---- host side -----------------------------------------------------------------------------------
CUtensorMapDataType tma_dtype(int dtype) {
  return dtype == MM_DTYPE_FLOAT ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                 : (dtype == MM_DTYPE_UINT8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16);
}
uint32_t elem_bytes(int dtype) { return dtype == MM_DTYPE_FLOAT ? 4u : (dtype == MM_DTYPE_UINT8 ? 1u : 2u); }

int encode(CUtensorMap *map, CUtensorMapDataType dt, const void *base, uint64_t inner, uint64_t outer, uint64_t pitch_bytes,
           uint32_t box_inner, uint32_t box_outer, CUtensorMapSwizzle swizzle, const char *what) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return fail(MM_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t gdim[2] = {inner, outer};
  cuuint64_t gstride[1] = {pitch_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, dt, 2, const_cast<void *>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    return fail(MM_ERR_CUDA, std::string("cuTensorMapEncodeTiled (") + what + ") failed with CUresult " +
                                 std::to_string(int(r)));
  }
  return MM_OK;
}

// K-major operand: `rows` rows of `k_elems` elements; box = {128 bytes of K, box_rows}, 128-byte
// swizzle, out-of-bounds reads return zeros (neutral for (Multiply, Add) — SURVEY.md section 5 trap 3).
int make_operand_map(CUtensorMap *map, const void *base, int dtype, uint64_t rows, uint64_t k_elems, uint32_t box_rows) {
  const uint32_t eb = elem_bytes(dtype);
  return encode(map, tma_dtype(dtype), base, k_elems, rows, k_elems * eb, uint32_t(BLOCK_K_BYTES / eb), box_rows,
                CU_TENSOR_MAP_SWIZZLE_128B, "K-major operand");
}

// C (`batch` packed row-major rows x m matrices) for the epilogue's TMA stores: 16 x 32 blocks,
// swizzle = row pitch of the block.  Three dimensions {m, rows, batch}, so that a block of a
// problem whose last rows are partial is clipped at that problem's end, not the batch's.
int make_c_map(CUtensorMap *map, void *base, int dtype, uint64_t rows, uint64_t m, uint64_t batch) {
  const uint32_t eb = elem_bytes(dtype);
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return fail(MM_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t gdim[3] = {m, rows, batch};
  cuuint64_t gstride[2] = {m * eb, rows * m * eb};
  cuuint32_t box[3] = {32, EPI_ROWS, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  const CUtensorMapSwizzle swizzle =
      eb == 4 ? CU_TENSOR_MAP_SWIZZLE_128B : (eb == 2 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
  CUresult r = enc(map, tma_dtype(dtype), 3, base, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    return fail(MM_ERR_CUDA, "cuTensorMapEncodeTiled (C) failed with CUresult " + std::to_string(int(r)));
  }
  return MM_OK;
}

int num_sms() {
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}

size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

template <typename T, bool ROUND>
void launch_transpose(const void *src, void *dst, uint32_t src_rows, uint32_t src_cols, cudaStream_t stream,
                      unsigned copies) {
  dim3 grid((src_cols + 63) / 64, (src_rows + 63) / 64, copies);
  transpose_prep_kernel<T, ROUND><<<grid, 256, 0, stream>>>(static_cast<const T *>(src), static_cast<T *>(dst),
                                                           src_rows, src_cols);
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

size_t tcgen05_bt_bytes(int dtype, unsigned k, unsigned m, int flags, const Tuning &t, unsigned b_copies) {
  if (tcgen05_b_in_place(dtype, flags, t)) return 0;
  const size_t eb = elem_bytes(dtype);
  return align_up(size_t(b_copies) * m * k * eb * (split3(dtype, flags) ? 3 : 1), 1024);
}

size_t tcgen05_scratch_bytes(int dtype, unsigned n, unsigned k, unsigned m, int flags, const Tuning &t,
                             const GemmBatch &batch) {
  const size_t eb = elem_bytes(dtype);
  size_t bytes = TAIL_BYTES + tcgen05_bt_bytes(dtype, k, m, flags, t, batch.b_copies());  // counters (tail) + B copies
  if (dtype == MM_DTYPE_FLOAT || (flags & MM_FLAG_TRANSPOSED_A)) {
    bytes += align_up(size_t(batch.a_copies()) * n * k * eb * (split3(dtype, flags) ? 3 : 1), 1024);
  }
  return bytes;
}

// Copy row-sliced B (slices on peer GPUs) into one local array: the NVLink all-gather of the
// multi-GPU path for the kernel families that consume B as stored.
int gather_b_rows(const BSource &src, void *dst, size_t elem_bytes, unsigned k, unsigned m, cudaStream_t stream) {
  return launch_panels(false, src, dst, elem_bytes, k, m, /*panel_cols=*/unsigned(1024 / elem_bytes), nullptr,
                       num_sms() * 2, stream);
}

int tcgen05_prepare_b(int dtype, const BSource &src, void *bt, unsigned k, unsigned m, int flags, const Tuning &t,
                      const void **b_op, unsigned int *ready, unsigned *ready_target, cudaStream_t stream,
                      unsigned copies) {
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
      MM_CUDA_TRY(cudaFuncSetAttribute(round_tf32_kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                                       cudaSharedmemCarveoutMaxShared));
      const size_t count4 = size_t(k) * m / 4;
      const int blocks = int(std::min<size_t>((count4 + 255) / 256, size_t(num_sms()) * 16));
      round_tf32_kernel<<<blocks, 256, 0, stream>>>(static_cast<const float4 *>(src.b), static_cast<float4 *>(bt), count4);
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
      launch_transpose<float, true>(b, bt, k, m, stream, copies);
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
// half A is used in place; A stored K x N (`transposed`, leading dimension = rows, only whole
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
    if (transposed) {
      if (t.tf32_no_round()) {
        launch_transpose<float, false>(a, aprep, k, rows, stream, copies);
      } else {
        launch_transpose<float, true>(a, aprep, k, rows, stream, copies);  // A stored K x N -> N x K
      }
      *a_op = aprep;
    } else if (!t.tf32_no_round()) {
      MM_CUDA_TRY(cudaFuncSetAttribute(round_tf32_kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                                       cudaSharedmemCarveoutMaxShared));  // see tcgen05_prepare_b
      const size_t count4 = all_rows * k / 4;
      const int blocks = int(std::min<size_t>((count4 + 255) / 256, size_t(num_sms()) * 16));
      round_tf32_kernel<<<blocks, 256, 0, stream>>>(static_cast<const float4 *>(a),
                                                   static_cast<float4 *>(aprep), count4);
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

struct LaunchPlan {
  const CUtensorMap *map_a, *map_b, *map_c;
  void *c;
  GemmParams p;
  int requested_stages;
  bool attributes_only;  // dry run: set the function attribute (loads the kernel), launch nothing
  cudaStream_t stream;
};

template <int KIND, typename TOut, int CG, int BN>
int launch_gemm_variant(LaunchPlan plan) {
  using G = Geo<CG, BN>;
  auto kern = gemm_wgmma_kernel<KIND, TOut, CG, BN>;
  // Ring depth: the deepest that fits unless the tuning asks for less.
  const int stages = plan.requested_stages <= 0 ? G::MAX_STAGES
                                                 : std::min(std::max(plan.requested_stages, 2), int(G::MAX_STAGES));
  const size_t smem = G::smem_bytes(stages);
  MM_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(G::smem_bytes(G::MAX_STAGES))));
  if (plan.attributes_only) return MM_OK;
  plan.p.num_stages = uint32_t(stages);
  plan.p.raster_group = std::max<uint32_t>(1u, plan.p.raster_group / G::TILE_ROWS);  // rows -> row tiles
  const uint32_t tiles = plan.p.batch * ceil_div(plan.p.rows, G::TILE_ROWS) * ceil_div(plan.p.cols, BN);
  const uint32_t groups = std::min<uint32_t>(tiles, uint32_t(num_sms()) / CG);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(groups * CG);
  cfg.blockDim = dim3(NUM_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = plan.stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CG;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if (plan.p.tile_sync) MM_CUDA_TRY(cudaMemsetAsync(plan.p.tile_sync, 0, sizeof(unsigned int), plan.stream));
  MM_CUDA_TRY(cudaLaunchKernelEx(&cfg, kern, *plan.map_a, *plan.map_b, *plan.map_c, static_cast<TOut *>(plan.c), plan.p));
  return MM_OK;
}

template <int KIND, typename TOut>
int dispatch_variant(int cg, int bn, const LaunchPlan &plan) {
#define MM_VARIANT(CGV, BNV) \
  if (cg == CGV && bn == BNV) return launch_gemm_variant<KIND, TOut, CGV, BNV>(plan);
  MM_VARIANT(2, 256)
  MM_VARIANT(1, 256)
  MM_VARIANT(2, 128)
  MM_VARIANT(1, 128)
#undef MM_VARIANT
  return fail(MM_ERR_INVALID, "no wgmma kernel variant for this tuning (cta_group 1|2, block_n 128|256)");
}

int gemm_dispatch(int dtype, const void *a_op, const void *b_op, void *c, unsigned rows, unsigned k, unsigned m,
                  int flags, const Tuning &t, unsigned int *tile_sync, const unsigned int *b_ready,
                  unsigned b_ready_target, bool attributes_only, cudaStream_t stream, const GemmBatch &batch) {
  if (split3(dtype, flags)) k *= 3;  // the operands carry [hi|hi|lo] x [hi|lo|hi] per 16-block of K
  const bool is_f32 = dtype == MM_DTYPE_FLOAT;
  const size_t eb = elem_bytes(dtype);
  const int cg = t.cta_group(), bn = t.block_n();
  if (batch.count > 1 && b_ready != nullptr) return fail(MM_ERR_UNSUPPORTED, "batched calls need a complete B operand");
  CUtensorMap map_a, map_b, map_c;
  std::memset(&map_c, 0, sizeof(map_c));
  LaunchPlan plan{&map_a, &map_b, &map_c, c, {}, t.stages(), attributes_only, stream};
  if (!attributes_only) {
    // the problems of a batch stacked along the rows (one copy when the operand is shared)
    int rc = make_operand_map(&map_a, a_op, dtype, uint64_t(batch.a_copies()) * rows, k, BLOCK_M);
    if (rc != MM_OK) return rc;
    rc = make_operand_map(&map_b, b_op, dtype, uint64_t(batch.b_copies()) * m, k, uint32_t(bn / cg));
    if (rc != MM_OK) return rc;
    if (t.tma_store()) {
      rc = make_c_map(&map_c, c, dtype, rows, m, batch.count);
      if (rc != MM_OK) return rc;
    }
  }
  plan.p.rows = rows;
  plan.p.cols = m;
  plan.p.batch = batch.count;
  plan.p.a_prob_rows = batch.shared_a ? 0u : rows;
  plan.p.b_prob_rows = batch.shared_b ? 0u : m;
  plan.p.k_bytes = uint32_t(size_t(k) * eb);
  plan.p.raster_group = uint32_t(std::max(1, t.raster_rows()));  // in rows here; per-variant tiles in the launcher
  plan.p.tma_store = t.tma_store() ? 1u : 0u;
  plan.p.b_ready_target = b_ready_target;
  plan.p.l2_policy = t.l2_policy() == 1 ? ptx::L2_EVICT_FIRST : (t.l2_policy() == 2 ? ptx::L2_EVICT_LAST : ptx::L2_EVICT_NORMAL);
  plan.p.tile_sync = t.tile_sync() ? tile_sync : nullptr;
  plan.p.b_ready = b_ready;
  if (dtype == MM_DTYPE_UINT8) return dispatch_variant<ptx::KIND_I8, unsigned char>(cg, bn, plan);
  return is_f32 ? dispatch_variant<ptx::KIND_TF32, float>(cg, bn, plan)
                : dispatch_variant<ptx::KIND_F16, __half>(cg, bn, plan);
}

}  // namespace

// C[rows x m] = Aop[rows x k] * B on the tensor cores; `b_op` as returned by tcgen05_prepare_b.
int tcgen05_gemm(int dtype, const void *a_op, const void *b_op, void *c, unsigned rows, unsigned k, unsigned m,
                 int flags, const Tuning &t, unsigned int *tile_sync, const unsigned int *b_ready,
                 unsigned b_ready_target, cudaStream_t stream, const GemmBatch &batch) {
  return gemm_dispatch(dtype, a_op, b_op, c, rows, k, m, flags, t, tile_sync, b_ready, b_ready_target, false, stream,
                       batch);
}

int tcgen05_prepare_b_async(int dtype, const BSource &src, void *local_b, void *scratch, size_t scratch_bytes,
                            unsigned k, unsigned m, int flags, const Tuning &t, cudaStream_t stream, cudaStream_t side,
                            cudaEvent_t ev_fork, cudaEvent_t ev_join, PreparedB *out, unsigned copies) {
  *out = PreparedB{};
  const bool in_place = tcgen05_b_in_place(dtype, flags, t);
  const bool parts = src.src != nullptr;
  if (copies != 1) {
    if (parts) return fail(MM_ERR_UNSUPPORTED, "batched calls take B from one array");
    return tcgen05_prepare_b(dtype, src, scratch, k, m, flags, t, &out->b_op, nullptr, nullptr, stream, copies);
  }
  if (parts && !tcgen05_b_mn(dtype, flags, t)) {
    // K-major copy requested (tuning / 3xTF32): assemble the slices first, then transpose locally
    int rc = gather_b_rows(src, local_b, elem_bytes(dtype), k, m, stream);
    if (rc != MM_OK) return rc;
    BSource whole;
    whole.b = local_b;
    return tcgen05_prepare_b(dtype, whole, scratch, k, m, flags, t, &out->b_op, nullptr, nullptr, stream);
  }
  void *bt = in_place ? local_b : scratch;
  const Tcgen05Counters cnt = tcgen05_counters(scratch, scratch_bytes);
  const unsigned panels = ceil_div(m, unsigned(t.block_n()));
  // the panel kernel runs (float rounding, or a gather of slices), a second stream exists, the tuning allows it
  const bool overlap = side != nullptr && t.b_overlap() != 0 && tcgen05_b_mn(dtype, flags, t) && (!in_place || parts) &&
                       panels <= B_READY_BYTES / sizeof(unsigned int);
  if (!overlap) return tcgen05_prepare_b(dtype, src, bt, k, m, flags, t, &out->b_op, nullptr, nullptr, stream);
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
  if (dtype != MM_DTYPE_FLOAT && dtype != MM_DTYPE_HALF && dtype != MM_DTYPE_UINT8) {
    return fail(MM_ERR_UNSUPPORTED, "tcgen05 path handles float, half and uint8_t only");
  }
  if (g.tuning == nullptr) return fail(MM_ERR_INVALID, "tcgen05 launch without tuning");
  const Tuning &t = *g.tuning;
  if (g.dry_run) {
    // force the lazily loaded kernels in (prep + the GEMM variant this tuning selects) and the driver entry point
    cudaFuncAttributes attr;
    MM_CUDA_TRY(cudaFuncGetAttributes(&attr, round_tf32_kernel));
    MM_CUDA_TRY(cudaFuncGetAttributes(&attr, prep_b_panels_kernel<true>));
    MM_CUDA_TRY(cudaFuncGetAttributes(&attr, prep_b_panels_kernel<false>));
    MM_CUDA_TRY(cudaFuncGetAttributes(&attr, transpose_prep_kernel<float, true>));
    MM_CUDA_TRY(cudaFuncGetAttributes(&attr, transpose_prep_kernel<__half, false>));
    MM_CUDA_TRY(cudaFuncGetAttributes(&attr, transpose_prep_kernel<unsigned char, false>));
    if (!get_encode_fn()) return fail(MM_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
    return gemm_dispatch(dtype, nullptr, nullptr, nullptr, g.n, g.k, g.m, g.flags, t, nullptr, nullptr, 0, true, g.stream,
                         g.batch);
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
  // one preparation pass per operand for the whole batch; a shared operand is prepared once
  int rc = tcgen05_prepare_b_async(dtype, src, nullptr, scratch, scratch_bytes, g.k, g.m, g.flags, t, g.stream,
                                   g.side_stream, g.ev_fork, g.ev_join, &pb, g.batch.b_copies());
  if (rc == MM_OK) rc = tcgen05_prepare_a(dtype, g.a, aprep, g.n, g.k, g.flags, t, &a_op, g.stream, g.batch.a_copies());
  if (rc == MM_OK && g.ev_prep_done) cudaEventRecord(g.ev_prep_done, g.stream);
  if (rc == MM_OK) {
    rc = tcgen05_gemm(dtype, a_op, pb.b_op, g.c, g.n, g.k, g.m, g.flags, t, cnt.tile_sync, pb.ready, pb.ready_target,
                      g.stream, g.batch);
  }
  if (pb.forked) cudaStreamWaitEvent(g.stream, g.ev_join, 0);  // join, on the error paths too
  return rc;
}

}  // namespace mm
