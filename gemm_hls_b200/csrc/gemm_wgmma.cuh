// The wgmma tensor-core GEMM kernel (C = A' * B'^T, both operands K-major) and its host-side launch
// machinery: tensor maps, run-time parameters and the per-variant launcher.  Shared by the translation
// units that instantiate it: gemm_tcgen05.cu (tf32, f16, u8), gemm_wgmma_bf16.cu (bf16), gemm_wgmma_b1.cu (bit-packed
// Boolean) and gemm_wgmma_acc.cu (the accumulate kernels of every type).  The kernel's
// structure is described at the top of gemm_tcgen05.cu.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <type_traits>

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
// Two adjacent accumulator values (columns c, c + 1 of one row) as the bytes of C.  The accumulate kernel
// (mm_kernel_enqueue_accumulate) then combines them with the old pair of C: add(old, p) = C_old + P, elementwise,
// in the type of C and with C_old as the first operand (load: ld.global, coherent with the kernel's own stores).
template <typename TOut>
struct Pair;
template <>
struct Pair<float> {
  using T = uint2;
  __device__ __forceinline__ static uint2 make(uint32_t a, uint32_t b) { return make_uint2(a, b); }
  __device__ __forceinline__ static uint2 load(const uint2 *p) {
    uint2 v;
    asm volatile("ld.global.v2.b32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p));
    return v;
  }
  __device__ __forceinline__ static uint2 add(uint2 old, uint2 p) {
    return make_uint2(__float_as_uint(__fadd_rn(__uint_as_float(old.x), __uint_as_float(p.x))),
                      __float_as_uint(__fadd_rn(__uint_as_float(old.y), __uint_as_float(p.y))));
  }
};
__device__ __forceinline__ uint32_t ld_global_b32(const uint32_t *p) {
  uint32_t v;
  asm volatile("ld.global.b32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}
template <>
struct Pair<__half> {
  using T = uint32_t;
  __device__ __forceinline__ static uint32_t make(uint32_t a, uint32_t b) {
    __half2 h = __floats2half2_rn(__uint_as_float(a), __uint_as_float(b));
    return *reinterpret_cast<uint32_t *>(&h);
  }
  __device__ __forceinline__ static uint32_t load(const uint32_t *p) { return ld_global_b32(p); }
  // HADD2: each half rounded exactly like the scalar __hadd_rn
  __device__ __forceinline__ static uint32_t add(uint32_t old, uint32_t p) {
    __half2 s = __hadd2_rn(*reinterpret_cast<__half2 *>(&old), *reinterpret_cast<__half2 *>(&p));
    return *reinterpret_cast<uint32_t *>(&s);
  }
};
// bfloat16: both accumulators rounded to nearest by one cvt.rn.bf16x2.f32.
template <>
struct Pair<__nv_bfloat16> {
  using T = uint32_t;
  __device__ __forceinline__ static uint32_t make(uint32_t a, uint32_t b) {
    __nv_bfloat162 h = __floats2bfloat162_rn(__uint_as_float(a), __uint_as_float(b));
    return *reinterpret_cast<uint32_t *>(&h);
  }
  __device__ __forceinline__ static uint32_t load(const uint32_t *p) { return ld_global_b32(p); }
  __device__ __forceinline__ static uint32_t add(uint32_t old, uint32_t p) {
    __nv_bfloat162 s = __hadd2_rn(*reinterpret_cast<__nv_bfloat162 *>(&old), *reinterpret_cast<__nv_bfloat162 *>(&p));
    return *reinterpret_cast<uint32_t *>(&s);
  }
};
// uint8_t: the accumulator is the exact 32-bit sum; its low byte is the reference's result (arithmetic modulo 256).
template <>
struct Pair<unsigned char> {
  using T = unsigned short;
  __device__ __forceinline__ static unsigned short make(uint32_t a, uint32_t b) {
    return static_cast<unsigned short>((a & 0xFFu) | ((b & 0xFFu) << 8));
  }
  __device__ __forceinline__ static unsigned short load(const unsigned short *p) {
    unsigned short v;
    asm volatile("ld.global.b16 %0, [%1];" : "=h"(v) : "l"(p));
    return v;
  }
  // two bytes, each added modulo 256
  __device__ __forceinline__ static unsigned short add(unsigned short old, unsigned short p) {
    const uint32_t lo = (uint32_t(old) + uint32_t(p)) & 0xFFu;
    const uint32_t hi = ((uint32_t(old) >> 8) + (uint32_t(p) >> 8)) & 0xFFu;
    return static_cast<unsigned short>(lo | (hi << 8));
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

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// Run-time launch parameters of the GEMM kernel (one struct so that the instantiations share a
// signature).
struct GemmParams {
  uint32_t rows, cols, k_bytes;
  uint32_t num_stages;       // ring depth actually used (<= Geo::MAX_STAGES, what the smem allocation holds)
  uint32_t raster_group;     // row tiles per rasterisation group
  uint32_t tma_store;        // 1: staged TMA-store epilogue, 0: direct stores
  // Batch: `batch` problems of rows x cols.  A and B are read through 2-D maps with the problems
  // stacked along the row dimension: problem i starts at row i * a_prob_rows of A and
  // i * b_prob_rows of B (0 = every problem reads the same operand).  C is a 3-D map {cols, rows, batch}.
  uint32_t batch, a_prob_rows, b_prob_rows;
  uint64_t l2_policy;
  unsigned int *tile_sync;        // soft wave-barrier counter or null
  // float only: per distinct A (B) operand of the batch, nonzero when every TF32-rounded value of it is exactly a half
  // (gemm_tcgen05.cu); a tile whose A and B both fit reads the fp16 copies and runs on the f16 wgmma.  Null: TF32 only.
  const unsigned int *fits_a, *fits_b;
};

// The counts of a b1 wgmma fragment (ptx::wgmma) as bits, count > 0: w[i][chunk] = columns 32 chunk .. + 32 of the
// lane's row i (of two), bit j % 32 for column j.  Each lane holds two columns of every eight of its rows; an OR over
// the four lanes of a row (q = lane % 4) assembles every word in all four.
template <int BN>
__device__ __forceinline__ void pack_bit_words(const uint32_t (&acc)[BN / 2], uint32_t q, uint32_t (&w)[2][BN / 32]) {
#pragma unroll
  for (int i = 0; i < 2; ++i) {
#pragma unroll
    for (int chunk = 0; chunk < BN / 32; ++chunk) {
      uint32_t x = 0;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
#pragma unroll
        for (int c = 0; c < 2; ++c) x |= uint32_t(acc[4 * (4 * chunk + j) + 2 * i + c] != 0u) << (8 * j + 2 * q + c);
      }
      x |= __shfl_xor_sync(0xFFFFFFFFu, x, 1);
      x |= __shfl_xor_sync(0xFFFFFFFFu, x, 2);
      w[i][chunk] = x;
    }
  }
}

// The 32 x 32 bit block whose row l is `x` in lane l becomes its transpose: bit c of lane l's word = bit l of lane c's
// word on entry.  Five exchange stages, each swapping the off-diagonal halves of every 2s x 2s sub-block.  Used by the
// b1 preparation (gemm_wgmma_b1.cu) and the Boolean closure (bool_closure.cu) to make row-major bits K-major.
__device__ __forceinline__ uint32_t warp_transpose32(uint32_t x, uint32_t lane) {
  uint32_t m = 0x0000FFFFu;
#pragma unroll
  for (int s = 16; s > 0; s >>= 1, m ^= m << s) {
    const uint32_t y = __shfl_xor_sync(0xFFFFFFFFu, x, s);
    x = (lane & s) ? ((x & ~m) | ((y >> s) & m)) : ((x & ~(m << s)) | ((y & m) << s));
  }
  return x;
}

// b1 epilogue (mm_kernel_enqueue_bool): this warp's 16 rows x BN columns of C as bits, C[i][j] = count > 0.  C rows
// are `cols` / 8 bytes; bit j % 8 of byte j / 8, least significant first.  A 128-column group of one row is 16
// bytes, the narrowest TMA box and one 128-bit store, so the warp writes whole groups: through the staging buffer
// and one TMA store of 16 rows x BN / 8 bytes (tma_store), or directly.
template <typename G, int BN>
__device__ __forceinline__ void store_bit_tile(const uint32_t (&acc)[BN / 2], const CUtensorMap &tmap_c,
                                               unsigned char *__restrict__ C, const GemmParams &p, const TileCoord &tc,
                                               uint32_t cta_rank, uint32_t cwarp, uint32_t lane, uint32_t buf) {
  constexpr int GROUPS = BN / 128;  // 128-column groups per row of the tile
  const uint32_t row0 = tc.r * G::TILE_ROWS + cta_rank * BLOCK_M + cwarp * EPI_ROWS;
  const uint32_t r_in = lane / 4, q = lane % 4;
  uint32_t w[2][BN / 32];
  pack_bit_words<BN>(acc, q, w);
  const uint32_t row_bytes = p.cols / 8;
  if (p.tma_store) {
    if (row0 >= p.rows) return;  // warp-uniform
    constexpr uint32_t PITCH = BN / 8;
    if (lane == 0) ptx::tma_store_wait_read<0>();  // the previous block has left the buffer
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 2; ++i) {
#pragma unroll
      for (int g = 0; g < GROUPS; ++g) {
        if (q == uint32_t(i * GROUPS + g)) {
          ptx::st_shared_v4(buf + (r_in + 8 * i) * PITCH + 16 * g, w[i][4 * g], w[i][4 * g + 1], w[i][4 * g + 2],
                            w[i][4 * g + 3]);
        }
      }
    }
    ptx::fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) {
      // clipped to rows x cols of this problem by the map
      ptx::tma_store_3d(&tmap_c, buf, int32_t(tc.c * (BN / 8)), int32_t(row0), int32_t(tc.prob));
      ptx::tma_store_commit();
    }
  } else {
    unsigned char *Cp = C + size_t(tc.prob) * p.rows * row_bytes;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const uint32_t row = row0 + r_in + 8 * i;
#pragma unroll
      for (int g = 0; g < GROUPS; ++g) {
        const uint32_t col = tc.c * BN + 128 * g;
        if (q == uint32_t(i * GROUPS + g) && row < p.rows && col < p.cols) {
          *reinterpret_cast<uint4 *>(Cp + size_t(row) * row_bytes + col / 8) =
              make_uint4(w[i][4 * g], w[i][4 * g + 1], w[i][4 * g + 2], w[i][4 * g + 3]);
        }
      }
    }
  }
}

// C[rows x cols] = A'[rows x k] * B'^T ; A' (rows x k) and B' (cols x k) K-major.  CG == 2 must be
// launched with cluster dimension (2, 1, 1).  ACC: C = C_old + A'B'^T, the add applied to the rounded product in
// the epilogue (gemm_wgmma_accumulate_kernel); nothing else differs.
// KIND_TF32 has two datapaths, chosen per tile from the problem's fits flags (GemmParams::fits_a / fits_b): the TF32
// operands through tmap_a / tmap_b and wgmma tf32, or their fp16 copies (the same values, exactly) through tmap_a16 /
// tmap_b16 and wgmma f16 at twice the issue rate.  A stage is 128 bytes of K either way: 32 floats or 64 halves.
template <int KIND, typename TOut, int CG, int BN, bool ACC>
__device__ __forceinline__ void gemm_wgmma_body(const CUtensorMap &tmap_a, const CUtensorMap &tmap_b,
                                                const CUtensorMap &tmap_a16, const CUtensorMap &tmap_b16,
                                                const CUtensorMap &tmap_c, TOut *__restrict__ C, const GemmParams &p) {
  using G = Geo<CG, BN>;
  // f16, bf16: 2; b1 moves its bits as bytes, as u8 does
  constexpr int ELEM_BYTES = (KIND == ptx::KIND_TF32) ? 4 : ((KIND == ptx::KIND_I8 || KIND == ptx::KIND_B1) ? 1 : 2);
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
  const uint32_t num_kb16 = (p.k_bytes / 2 + BLOCK_K_BYTES - 1) / BLOCK_K_BYTES;  // the fp16 copies: half the bytes
  // both roles of the CTA take the same datapath for a tile: the producer loads what the consumers multiply
  auto half_tile = [&](const TileCoord &tc) -> bool {
    if constexpr (KIND != ptx::KIND_TF32) return false;
    if (p.fits_a == nullptr) return false;
    return p.fits_a[p.a_prob_rows ? tc.prob : 0u] != 0u && p.fits_b[p.b_prob_rows ? tc.prob : 0u] != 0u;
  };

  if (threadIdx.x == 0) {
    ptx::prefetch_tensormap(&tmap_a);
    ptx::prefetch_tensormap(&tmap_b);
    if (p.tma_store) ptx::prefetch_tensormap(&tmap_c);
    if (KIND == ptx::KIND_TF32 && p.fits_a != nullptr) {
      ptx::prefetch_tensormap(&tmap_a16);
      ptx::prefetch_tensormap(&tmap_b16);
    }
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
        const bool h = half_tile(tc);
        const CUtensorMap *map_a = h ? &tmap_a16 : &tmap_a;
        const CUtensorMap *map_b = h ? &tmap_b16 : &tmap_b;
        const uint32_t tile_kb = h ? num_kb16 : num_kb;
        const int32_t kb_elems = h ? BLOCK_K_BYTES / 2 : BLOCK_K_ELEMS;
        for (uint32_t kb = 0; kb < tile_kb; ++kb) {
          ptx::mbar_wait(empty_bar(stage), phase ^ 1);
          const uint32_t sa = smem_a0 + stage * G::A_STAGE_BYTES;
          const uint32_t sb = smem_b0 + stage * G::B_STAGE_BYTES + cta_rank * G::LOAD_N * BLOCK_K_BYTES;
          const int32_t k0 = kb * kb_elems;
          ptx::mbar_arrive_expect_tx(full_bar(stage), G::STAGE_BYTES);
          ptx::tma_load_2d(sa, map_a, full_bar(stage), k0, a_row, p.l2_policy);
          if (CG == 1) {
            ptx::tma_load_2d(sb, map_b, full_bar(stage), k0, b_row, p.l2_policy);
          } else {
            ptx::tma_load_2d_multicast(sb, map_b, full_bar(stage), k0, b_row, 0x3, p.l2_policy);
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
      // The k-loop once per datapath, each a whole wgmma pipeline up to its final wait: a branch between the issue
      // and the wait of one pipeline would make ptxas serialise every wgmma.
      auto mainloop = [&](auto kind, uint32_t tile_kb) {
        uint32_t prev = 0;
        for (uint32_t kb = 0; kb < tile_kb; ++kb) {
          ptx::mbar_wait(full_bar(stage), phase);
          const uint64_t adesc = ptx::make_smem_desc_k_sw128(smem_a0 + stage * G::A_STAGE_BYTES + wg * 64 * BLOCK_K_BYTES);
          const uint64_t bdesc = ptx::make_smem_desc_k_sw128(smem_b0 + stage * G::B_STAGE_BYTES);
          ptx::wgmma_fence();
#pragma unroll
          for (int k = 0; k < BLOCK_K_BYTES / WGMMA_K_BYTES; ++k) {
            ptx::wgmma<decltype(kind)::value, BN>(acc, adesc + uint64_t(k * (WGMMA_K_BYTES >> 4)),
                                                  bdesc + uint64_t(k * (WGMMA_K_BYTES >> 4)),
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
      };
      if (KIND == ptx::KIND_TF32 && half_tile(tc)) {
        mainloop(std::integral_constant<int, ptx::KIND_F16>{}, num_kb16);
      } else {
        mainloop(std::integral_constant<int, KIND>{}, num_kb);
      }

      if constexpr (KIND == ptx::KIND_B1) {
        store_bit_tile<G, BN>(acc, tmap_c, C, p, tc, cta_rank, cwarp, lane, buf);
        continue;
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
            typename P::T old[4][2];
            if constexpr (ACC) {
              // C_old of this lane's pairs, all eight loads in flight before the first is used; pairs outside
              // the problem are not read (the TMA store clips them)
              const TOut *Cp = C + size_t(tc.prob) * rows * cols;
#pragma unroll
              for (int j = 0; j < 4; ++j) {
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                  const uint32_t row = row0 + r_in + 8 * i, c = col + 8 * j + c_in;
                  old[j][i] = typename P::T{};
                  if (row < rows && c < cols) {
                    old[j][i] = P::load(reinterpret_cast<const typename P::T *>(Cp + size_t(row) * cols + c));
                  }
                }
              }
            }
            if (lane == 0) ptx::tma_store_wait_read<0>();         // the previous block has left the buffer
            __syncwarp();
#pragma unroll
            for (int j = 0; j < 4; ++j) {
#pragma unroll
              for (int i = 0; i < 2; ++i) {
                const uint32_t a = buf + (r_in + 8 * i) * PITCH + (8 * j + c_in) * sizeof(TOut);
                const int reg = 4 * (4 * chunk + j) + 2 * i;
                typename P::T v = P::make(acc[reg], acc[reg + 1]);
                if constexpr (ACC) v = P::add(old[j][i], v);
                st_shared_pair(a ^ (((a >> 7) & SW_MASK) << 4), v);
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
          if constexpr (ACC) {
            // groups of eight pairs: eight loads of C_old in flight, then eight stores
#pragma unroll
            for (int j0 = 0; j0 < BN / 8; j0 += 8) {
              typename P::T old[8];
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                const uint32_t col = tc.c * BN + 8 * (j0 + j) + c_in;
                old[j] = typename P::T{};
                if (col < cols) old[j] = P::load(crow + col / 2);
              }
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                const uint32_t col = tc.c * BN + 8 * (j0 + j) + c_in;
                const int reg = 4 * (j0 + j) + 2 * i;
                if (col < cols) crow[col / 2] = P::add(old[j], P::make(acc[reg], acc[reg + 1]));
              }
            }
          } else {
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
              const uint32_t col = tc.c * BN + 8 * j + c_in;
              if (col < cols) crow[col / 2] = P::make(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]);
            }
          }
        }
      }
    }
    if (p.tma_store && lane == 0) ptx::tma_store_wait_all<0>();  // stores complete before the CTA's smem goes away
  }

  // no CTA of a cluster leaves while its peer may still multicast into it or arrive on its barriers
  if (CG == 2) cluster_sync_all();
}

template <int KIND, typename TOut, int CG, int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                  const __grid_constant__ CUtensorMap tmap_a16, const __grid_constant__ CUtensorMap tmap_b16,
                  const __grid_constant__ CUtensorMap tmap_c, TOut *__restrict__ C, const GemmParams p) {
  gemm_wgmma_body<KIND, TOut, CG, BN, false>(tmap_a, tmap_b, tmap_a16, tmap_b16, tmap_c, C, p);
}

// C <- C + A'B'^T (mm_kernel_enqueue_accumulate); instantiated in gemm_wgmma_acc.cu only.
template <int KIND, typename TOut, int CG, int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_wgmma_accumulate_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                             const __grid_constant__ CUtensorMap tmap_a16, const __grid_constant__ CUtensorMap tmap_b16,
                             const __grid_constant__ CUtensorMap tmap_c, TOut *__restrict__ C, const GemmParams p) {
  gemm_wgmma_body<KIND, TOut, CG, BN, true>(tmap_a, tmap_b, tmap_a16, tmap_b16, tmap_c, C, p);
}

// ---- host side -----------------------------------------------------------------------------------
CUtensorMapDataType tma_dtype(int dtype) {
  if (dtype == MM_DTYPE_BFLOAT16) return CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
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

struct LaunchPlan {
  const CUtensorMap *map_a, *map_b, *map_c;
  const CUtensorMap *map_a16, *map_b16;  // float's fp16 operand copies; map_a / map_b again for the other types
  void *c;
  GemmParams p;
  int requested_stages;
  bool attributes_only;  // dry run: set the function attribute (loads the kernel), launch nothing
  cudaStream_t stream;
};

// Only the kernel a translation unit launches is instantiated there.
template <int KIND, typename TOut, int CG, int BN, bool ACC>
constexpr auto gemm_kernel_ptr() {
  if constexpr (ACC) return gemm_wgmma_accumulate_kernel<KIND, TOut, CG, BN>;
  else return gemm_wgmma_kernel<KIND, TOut, CG, BN>;
}

template <int KIND, typename TOut, int CG, int BN, bool ACC>
int launch_gemm_variant(LaunchPlan plan) {
  using G = Geo<CG, BN>;
  auto kern = gemm_kernel_ptr<KIND, TOut, CG, BN, ACC>();
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
  MM_CUDA_TRY(cudaLaunchKernelEx(&cfg, kern, *plan.map_a, *plan.map_b, *plan.map_a16, *plan.map_b16, *plan.map_c,
                                 static_cast<TOut *>(plan.c), plan.p));
  return MM_OK;
}

// ACC: the accumulate kernels (gemm_wgmma_acc.cu)
template <int KIND, typename TOut, bool ACC = false>
int dispatch_variant(int cg, int bn, const LaunchPlan &plan) {
#define MM_VARIANT(CGV, BNV) \
  if (cg == CGV && bn == BNV) return launch_gemm_variant<KIND, TOut, CGV, BNV, ACC>(plan);
  MM_VARIANT(2, 256)
  MM_VARIANT(1, 256)
  MM_VARIANT(2, 128)
  MM_VARIANT(1, 128)
#undef MM_VARIANT
  return fail(MM_ERR_INVALID, "no wgmma kernel variant for this tuning (cta_group 1|2, block_n 128|256)");
}

// The tensor maps and run-time parameters of one GEMM launch: everything but the kernel variant.  `maps`
// (A, B, C, fp16 A, fp16 B) must outlive the launch; `k` is the K extent the operands carry.  `half`: float's fp16
// operand copies and fits flags (gemm_tcgen05.cu), or empty.
int plan_gemm(int dtype, const void *a_op, const void *b_op, void *c, unsigned rows, unsigned k, unsigned m,
              const Tuning &t, unsigned int *tile_sync, bool attributes_only, cudaStream_t stream,
              const GemmBatch &batch, const HalfOperands &half, CUtensorMap (&maps)[5], LaunchPlan *plan) {
  const size_t eb = elem_bytes(dtype);
  const int cg = t.cta_group(), bn = t.block_n();
  const bool use_half = dtype == MM_DTYPE_FLOAT && half.fits_a != nullptr;
  std::memset(&maps[2], 0, sizeof(maps[2]));
  *plan = LaunchPlan{&maps[0], &maps[1], &maps[2], use_half ? &maps[3] : &maps[0], use_half ? &maps[4] : &maps[1],
                     c, {}, t.stages(), attributes_only, stream};
  if (!attributes_only) {
    // the problems of a batch stacked along the rows (one copy when the operand is shared)
    int rc = make_operand_map(&maps[0], a_op, dtype, uint64_t(batch.a_copies()) * rows, k, BLOCK_M);
    if (rc != MM_OK) return rc;
    rc = make_operand_map(&maps[1], b_op, dtype, uint64_t(batch.b_copies()) * m, k, uint32_t(bn / cg));
    if (rc != MM_OK) return rc;
    if (use_half) {
      rc = make_operand_map(&maps[3], half.a, MM_DTYPE_HALF, uint64_t(batch.a_copies()) * rows, k, BLOCK_M);
      if (rc != MM_OK) return rc;
      rc = make_operand_map(&maps[4], half.b, MM_DTYPE_HALF, uint64_t(batch.b_copies()) * m, k, uint32_t(bn / cg));
      if (rc != MM_OK) return rc;
    }
    if (t.tma_store()) {
      rc = make_c_map(&maps[2], c, dtype, rows, m, batch.count);
      if (rc != MM_OK) return rc;
    }
  }
  GemmParams &p = plan->p;
  p.rows = rows;
  p.cols = m;
  p.batch = batch.count;
  p.a_prob_rows = batch.shared_a ? 0u : rows;
  p.b_prob_rows = batch.shared_b ? 0u : m;
  p.k_bytes = uint32_t(size_t(k) * eb);
  p.raster_group = uint32_t(std::max(1, t.raster_rows()));  // in rows here; per-variant tiles in the launcher
  p.tma_store = t.tma_store() ? 1u : 0u;
  p.l2_policy = t.l2_policy() == 1 ? ptx::L2_EVICT_FIRST : (t.l2_policy() == 2 ? ptx::L2_EVICT_LAST : ptx::L2_EVICT_NORMAL);
  p.tile_sync = t.tile_sync() ? tile_sync : nullptr;
  p.fits_a = use_half ? half.fits_a : nullptr;
  p.fits_b = use_half ? half.fits_b : nullptr;
  return MM_OK;
}

}  // namespace

// bf16 (Multiply, Add): the four bf16 instantiations of the kernel live in their own translation unit,
// gemm_wgmma_bf16.cu.  Arguments as gemm_dispatch in gemm_tcgen05.cu.
int wgmma_bf16_gemm(const void *a_op, const void *b_op, void *c, unsigned rows, unsigned k, unsigned m, const Tuning &t,
                    unsigned int *tile_sync, bool attributes_only, cudaStream_t stream, const GemmBatch &batch);

// C <- C + product for every type of the wgmma path (mm_kernel_enqueue_accumulate): the sixteen accumulate kernels
// live in gemm_wgmma_acc.cu.  `k` is the K extent the operands carry (3K for 3xTF32).
int wgmma_accumulate_gemm(int dtype, const void *a_op, const void *b_op, void *c, unsigned rows, unsigned k, unsigned m,
                          const Tuning &t, unsigned int *tile_sync, bool attributes_only, cudaStream_t stream,
                          const GemmBatch &batch, const HalfOperands &half);

}  // namespace mm
