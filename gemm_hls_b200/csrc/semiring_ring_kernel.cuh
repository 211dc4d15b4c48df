// Ring variant of the CUDA-core semiring tile kernel for 4-byte element types with A stored row-major:
// BOTH tiles arrive by TMA into a 4-stage ring, stages are handed over through mbarriers (full: TMA
// transaction bytes; empty: one arrival per warp), and there is no block-wide barrier in the main loop.
//
// Why: what separates semiring_tile_kernel from its inner loop alone is the per-k-tile __syncthreads (every 16
// k-steps), the LDG + transposing STS of the A tile and its address arithmetic, and the 8 staging
// registers.  The variant's step is the tile body's, so the per-element order of operations is the same (bit-exact).
//
// Layout.  B tile: [16 k][128 columns], dense, as before.  A tile: [128 rows][16 k] = dense 64-byte rows, as
// it lies in HBM (no transposition); one LDS.128 yields four consecutive k of one row, so the eight rows of a
// thread cost eight LDS.128 per four k-steps — the same count as the k-major tile of semiring_tile_kernel.
// The sixteen lanes of a half-warp share ty, i.e. every 8-lane phase of an LDS.128 reads ONE address
// (broadcast): the A loads are conflict-free without any swizzle; the B loads are as before.
#pragma once

#include <cuda_runtime.h>

#include <type_traits>

#include "ptx_sm90.cuh"
#include "semiring.cuh"
#include "tma_host.cuh"

namespace mm {

struct SemiringRing {
  static constexpr int BM = 128, BN = 128, BK = 16;  // BK elements of 4 bytes = one 64-byte memory word
  static constexpr int STAGES = 4;
  // Tiles are requested AHEAD = STAGES - 2 iterations early: the stage being refilled in iteration kt held
  // tile kt - 2, which every warp released at least one iteration ago — the issuing thread does not have to
  // wait for the slowest warp of the previous tile, so warps may drift by a whole tile.
  static constexpr int AHEAD = STAGES - 2;
  static constexpr int THREADS = 256;
  static constexpr uint32_t A_BYTES = BM * BK * 4, B_BYTES = BK * BN * 4, STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr size_t SMEM_BYTES = size_t(STAGES) * STAGE_BYTES + 2 * STAGES * 8 + 1024;
};

// The TMA-ring main loop.  Both maps hold the problems stacked along their rows: problem blockIdx.z's A tile starts
// at row blockIdx.z * a_step * size_n + row0, column a_k0 (a tile of A may run past N into the next problem: those
// rows of C are never stored); its B tiles at row blockIdx.z * b_step * b_rows + b_k0, column col0 (a tile of B never
// crosses a problem: K % BK == 0).  The loop covers B's rows from b_k0 to the end of the problem (b_rows), at most
// V::kMaxK of them: a multiple of BK.
template <class V>
__device__ __forceinline__ void semiring_ring_body(V &&v, const CUtensorMap &tmap_a, unsigned a_step, unsigned a_k0,
                                                   const CUtensorMap &tmap_b, unsigned b_step, unsigned b_rows,
                                                   unsigned b_k0) {
  using T = typename V::T;
  using Reduce = typename V::Reduce;
  using Term = typename V::Term;
  static_assert(sizeof(T) == 4, "ring variant: 4-byte element types");
  static_assert(V::TN == 8, "ring variant: 8 x 8 elements per thread");
  using Cfg = SemiringRing;
  constexpr int BM = Cfg::BM, BN = Cfg::BN, BK = Cfg::BK, STAGES = Cfg::STAGES;
  const unsigned size_n = v.size_n, size_m = v.size_m;
  T *C = v.C + size_t(blockIdx.z) * size_n * size_m;
  const unsigned a_row0 = blockIdx.z * a_step * size_n, b_row0 = blockIdx.z * b_step * b_rows;

  extern __shared__ unsigned char smem_raw[];
  const uint32_t smem0 = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t full0 = smem0 + STAGES * Cfg::STAGE_BYTES, empty0 = full0 + 8 * STAGES;

  const int tid = threadIdx.x, lane = tid % 32;
  const int tx = tid % 16;  // column quad index
  const int ty = tid / 16;  // row quad index
  const unsigned row0 = blockIdx.y * BM, col0 = blockIdx.x * BN;
  const unsigned k_tiles = min(b_rows - b_k0, V::kMaxK) / BK;

  if (tid == 0) {
    ptx::prefetch_tensormap(&tmap_a);
    ptx::prefetch_tensormap(&tmap_b);
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(full0 + 8 * s, 1);
      ptx::mbar_init(empty0 + 8 * s, Cfg::THREADS / 32);
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();

  // tile kt -> stage kt % STAGES (thread 0 only).  A refill waits until all eight warps have released
  // the stage; see AHEAD for why that wait is normally already satisfied.
  auto load_tile = [&](unsigned kt) {
    const int stage = kt % STAGES;
    if (kt >= STAGES) ptx::mbar_wait(empty0 + 8 * stage, ((kt / STAGES) - 1) & 1);
    const uint32_t as = smem0 + stage * Cfg::STAGE_BYTES, bs = as + Cfg::A_BYTES, bar = full0 + 8 * stage;
    ptx::mbar_arrive_expect_tx(bar, Cfg::STAGE_BYTES);
    ptx::tma_load_2d(as, &tmap_a, bar, int32_t(a_k0 + kt * BK), int32_t(a_row0 + row0), ptx::L2_EVICT_NORMAL);
    ptx::tma_load_2d(bs, &tmap_b, bar, int32_t(col0), int32_t(b_row0 + b_k0 + kt * BK), ptx::L2_EVICT_NORMAL);
  };
  if (tid == 0) {
    for (unsigned kt = 0; kt < unsigned(Cfg::AHEAD) && kt < k_tiles; ++kt) load_tile(kt);
  }

  T acc[8][8];
  typename V::State state[8][8];
  v.seed(acc, state, C, row0, col0, tx, ty);

  const int r_lo = ty * 4, r_hi = 64 + ty * 4;  // this thread's rows: r_lo .. r_lo + 3 and r_hi .. r_hi + 3

  for (unsigned kt = 0; kt < k_tiles; ++kt) {
    const int stage = kt % STAGES;
    if (tid == 0 && kt + Cfg::AHEAD < k_tiles) load_tile(kt + Cfg::AHEAD);
    ptx::mbar_wait(full0 + 8 * stage, (kt / STAGES) & 1);
    const unsigned char *as = smem_raw + (smem0 - ptx::smem_u32(smem_raw)) + stage * Cfg::STAGE_BYTES;
    const T *bs = reinterpret_cast<const T *>(as + Cfg::A_BYTES);

#pragma unroll
    for (int c = 0; c < BK / 4; ++c) {  // four k per 16-byte chunk of an A row
      T a4[8][4];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int r = (i < 4 ? r_lo : r_hi) + (i % 4);
        const Quad<T> q = *reinterpret_cast<const Quad<T> *>(as + r * 64 + c * 16);
#pragma unroll
        for (int u = 0; u < 4; ++u) a4[i][u] = Term::prep(q.v[u]);
      }
#pragma unroll
      for (int kp = 0; kp < 4; kp += 2) {  // two consecutive k per step, reduced in order (see SemiringVariant::step)
        const int kk = c * 4 + kp;
        T bf[2][8];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const Quad<T> b0 = *reinterpret_cast<const Quad<T> *>(bs + (kk + u) * BN + tx * 4);
          const Quad<T> b1 = *reinterpret_cast<const Quad<T> *>(bs + (kk + u) * BN + 64 + tx * 4);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            bf[u][q] = Term::prep(b0.v[q]);
            bf[u][4 + q] = Term::prep(b1.v[q]);
          }
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            acc[i][j] = v.step(acc[i][j], state[i][j], a4[i][kp], bf[0][j], a4[i][kp + 1], bf[1][j], kt * BK + kk);
          }
        }
      }
    }
    __syncwarp();
    if (lane == 0) ptx::mbar_arrive(empty0 + 8 * stage);  // this warp is done reading the stage
  }

  if constexpr (V::kFinish) {
    v.finish(acc, state, row0, col0, tx, ty);
  } else {
    // Write the C tile once, masked to n < N, m < M (the role of WriteC, kernel/Memory.cpp:361-392).
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const size_t row = size_t(row0) + (i / 4) * 64 + ty * 4 + (i % 4);
      if (row >= size_n) continue;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const size_t col = size_t(col0) + h * 64 + tx * 4;
        if (col + 4 <= size_m) {
          Quad<T> out;
#pragma unroll
          for (int q = 0; q < 4; ++q) out.v[q] = acc[i][h * 4 + q];
          if constexpr (V::kAccumulate) {
            const Quad<T> old = *reinterpret_cast<const Quad<T> *>(C + row * size_m + col);
#pragma unroll
            for (int q = 0; q < 4; ++q) out.v[q] = Reduce::Apply(old.v[q], out.v[q]);
          }
          *reinterpret_cast<Quad<T> *>(C + row * size_m + col) = out;
        }
      }
    }
  }
}

template <typename T, class Map, class Reduce, bool ACC>
__device__ __forceinline__ void semiring_ring_product(const CUtensorMap &tmap_a, const CUtensorMap &tmap_b,
                                                      T *__restrict__ C, unsigned size_n, unsigned size_k,
                                                      unsigned size_m, unsigned a_step, unsigned b_step) {
  semiring_ring_body(SemiringVariant<T, Map, Reduce, ACC>{C, size_n, size_m}, tmap_a, a_step, 0u, tmap_b, b_step,
                     size_k, 0u);
}

template <typename T, class Map, class Reduce>
__global__ void __launch_bounds__(256, 2)
semiring_ring_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                     T *__restrict__ C, unsigned size_n, unsigned size_k, unsigned size_m, unsigned a_step,
                     unsigned b_step) {
  semiring_ring_product<T, Map, Reduce, false>(tmap_a, tmap_b, C, size_n, size_k, size_m, a_step, b_step);
}

// C <- Reduce(C_old, A (x) B) (mm_kernel_enqueue_accumulate); instantiated by semiring_accumulate_inst.cu only.
template <typename T, class Map, class Reduce>
__global__ void __launch_bounds__(256, 2)
semiring_accumulate_ring_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                                T *__restrict__ C, unsigned size_n, unsigned size_k, unsigned size_m, unsigned a_step,
                                unsigned b_step) {
  semiring_ring_product<T, Map, Reduce, true>(tmap_a, tmap_b, C, size_n, size_k, size_m, a_step, b_step);
}

}  // namespace mm
