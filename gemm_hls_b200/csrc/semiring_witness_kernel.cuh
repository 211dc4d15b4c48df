// Witness variants of the CUDA-core semiring kernels (mm_kernel_enqueue_witness): C exactly as
// semiring_tile_kernel / semiring_ring_kernel compute it, and beside every accumulator a uint32 register holding
// the last k at which the Min / Max reduction selected its new term (MM_WITNESS_NONE if it never did).
//
// Same tiles, same staging and the same per-element order of operations as the plain kernels: each step computes
// t = Map(a, b) once, decides Selects<Reduce>::apply(acc, t), applies Reduce::Apply(acc, t) (FMNMX stays FMNMX on
// the float default, so C keeps its bits) and moves k into the witness when the term was selected.  The two k of an
// unrolled pair are processed in order, k then k + 1, as Naive<> does.
//
// Registers: the witnesses double the accumulator file, so both kernels run one CTA (8 warps) per SM.  The ring
// kernel keeps 8 x 8 elements per thread (64 accumulators + 64 witnesses); the register-staged kernel, which also
// holds the next A tile in registers, keeps 8 x 4 (a 128 x 64 CTA tile) and does not unroll its k loop, so that no
// instantiation spills (ptxas hoists the data-independent terms of an unrolled And Map far enough ahead to).
#pragma once

#include <cuda_runtime.h>

#include <cstdint>

#include "common.cuh"
#include "semiring_kernel.cuh"

namespace mm {

// Register-staged witness kernel: every type, A row-major or stored K x N.  A as in semiring_tile_kernel (through
// registers, transposed into shared memory); B by TMA, BK rows x BN columns.
template <typename T>
struct WitnessTile {
  static constexpr int TN = 4;  // columns per thread: one quad
  static constexpr int BM = 128, BN = 16 * TN;
  static constexpr int BK = SemiringTile<T>::BK, VEC = SemiringTile<T>::VEC, LDA = SemiringTile<T>::LDA;
  static constexpr int THREADS = 256;
  static constexpr int CHUNKS_PER_THREAD = SemiringTile<T>::CHUNKS_PER_THREAD;  // A: 128 x 64 B = 512 chunks
  static constexpr int A_CHUNKS_PER_ROW = BK / VEC;                             // row-major A: per row of A
  static constexpr int AT_CHUNKS_PER_ROW = BM / VEC;                            // A stored K x N: per k
  static constexpr size_t A_BYTES = SemiringTile<T>::A_BYTES;
  static constexpr size_t B_TILE_BYTES = size_t(BK) * BN * sizeof(T);
  static constexpr size_t SMEM_BYTES = A_BYTES + 2 * B_TILE_BYTES + 16;
};

// One element-step: t = Map(a, b); the witness takes k when Reduce selects t.
template <class Map, class Reduce, typename T>
__device__ __forceinline__ void witness_step(T &acc, unsigned &w, T a, T b, unsigned k) {
  const T t = Map::Apply(a, b);
  const bool s = Selects<Reduce>::apply(acc, t);
  acc = Reduce::Apply(acc, t);
  w = s ? k : w;
}

// Rows i (0..7) and columns j (0..TN-1) of a thread's tile within the CTA tile, as in the plain kernels.
__device__ __forceinline__ int witness_row(int i, int ty) { return (i / 4) * 64 + ty * 4 + (i % 4); }
__device__ __forceinline__ int witness_col(int j, int tx) { return (j / 4) * 64 + tx * 4 + (j % 4); }

template <typename T, int TN>
__device__ __forceinline__ void witness_epilogue(const T (&acc)[8][TN], const unsigned (&wit)[8][TN], T *C,
                                                 unsigned *W, size_t row0, size_t col0, int tx, int ty,
                                                 unsigned size_n, unsigned size_m) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const size_t row = row0 + witness_row(i, ty);
    if (row >= size_n) continue;
#pragma unroll
    for (int h = 0; h < TN / 4; ++h) {
      const size_t col = col0 + witness_col(4 * h, tx);
      if (col + 4 <= size_m) {
        Quad<T> out;
#pragma unroll
        for (int q = 0; q < 4; ++q) out.v[q] = acc[i][h * 4 + q];
        *reinterpret_cast<Quad<T> *>(C + row * size_m + col) = out;
        *reinterpret_cast<uint4 *>(W + row * size_m + col) =
            make_uint4(wit[i][h * 4], wit[i][h * 4 + 1], wit[i][h * 4 + 2], wit[i][h * 4 + 3]);
      }
    }
  }
}

template <typename T, class Map, class Reduce>
__global__ void __launch_bounds__(256, 1)
semiring_witness_tile_kernel(const T *__restrict__ A, const __grid_constant__ CUtensorMap tmap_b, T *__restrict__ C,
                             unsigned *__restrict__ W, unsigned size_n, unsigned size_k, unsigned size_m,
                             bool TRANSPOSED_A, unsigned a_step, unsigned b_step) {
  using Cfg = WitnessTile<T>;
  constexpr int BM = Cfg::BM, BN = Cfg::BN, BK = Cfg::BK, VEC = Cfg::VEC, TN = Cfg::TN;
  constexpr int LDA = Cfg::LDA;
  A += size_t(blockIdx.z * a_step) * size_n * size_k;
  C += size_t(blockIdx.z) * size_n * size_m;
  W += size_t(blockIdx.z) * size_n * size_m;
  const unsigned b_k0 = blockIdx.z * b_step * size_k;  // first row of this problem's B in the map

  extern __shared__ __align__(128) unsigned char smem_raw[];
  T *As = reinterpret_cast<T *>(smem_raw);                 // [2][BK][LDA]  (k-major: A transposed)
  T *Bs = reinterpret_cast<T *>(smem_raw + Cfg::A_BYTES);  // [2][BK][BN]   (TMA destination)
  const uint32_t bar0 = ptx::smem_u32(smem_raw + Cfg::A_BYTES + 2 * Cfg::B_TILE_BYTES);  // full[0], full[1]

  const int tid = threadIdx.x;
  const int tx = tid % 16;  // column quad index
  const int ty = tid / 16;  // row quad index
  const size_t row0 = size_t(blockIdx.y) * BM;
  const size_t col0 = size_t(blockIdx.x) * BN;

  T acc[8][TN];
  unsigned wit[8][TN];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      acc[i][j] = Reduce::identity();
      wit[i][j] = MM_WITNESS_NONE;
    }
  }

  Chunk16<T> a_stage[Cfg::CHUNKS_PER_THREAD];

  if (tid == 0) {
    ptx::prefetch_tensormap(&tmap_b);
    ptx::mbar_init(bar0, 1);
    ptx::mbar_init(bar0 + 8, 1);
    ptx::fence_mbar_init();
  }
  __syncthreads();
  auto load_b_tma = [&](int buf, unsigned k0) {
    if (tid == 0) {
      ptx::mbar_arrive_expect_tx(bar0 + 8 * buf, uint32_t(Cfg::B_TILE_BYTES));
      ptx::tma_load_2d(ptx::smem_u32(Bs + buf * BK * BN), &tmap_b, bar0 + 8 * buf, int32_t(col0), int32_t(b_k0 + k0),
                       ptx::L2_EVICT_NORMAL);
    }
  };

  auto load_global = [&](unsigned k0) {
#pragma unroll
    for (int i = 0; i < Cfg::CHUNKS_PER_THREAD; ++i) {
      const int c = tid + i * Cfg::THREADS;
      if (!TRANSPOSED_A) {
        const int r = c / Cfg::A_CHUNKS_PER_ROW;
        const int part = c % Cfg::A_CHUNKS_PER_ROW;
        size_t row = row0 + r;
        if (row >= size_n) row = size_n - 1;  // clamp: rows past N are computed but never stored
        a_stage[i] = *reinterpret_cast<const Chunk16<T> *>(A + row * size_k + k0 + part * VEC);
      } else {
        const int kk = c / Cfg::AT_CHUNKS_PER_ROW;
        const int part = c % Cfg::AT_CHUNKS_PER_ROW;
#pragma unroll
        for (int v = 0; v < VEC; ++v) {
          size_t row = row0 + part * VEC + v;
          if (row >= size_n) row = size_n - 1;
          a_stage[i].v[v] = A[size_t(k0 + kk) * size_n + row];
        }
      }
    }
  };

  auto store_shared = [&](int buf) {
    T *as = As + buf * BK * LDA;
#pragma unroll
    for (int i = 0; i < Cfg::CHUNKS_PER_THREAD; ++i) {
      const int c = tid + i * Cfg::THREADS;
      if (!TRANSPOSED_A) {
        const int r = c / Cfg::A_CHUNKS_PER_ROW;
        const int part = c % Cfg::A_CHUNKS_PER_ROW;
#pragma unroll
        for (int v = 0; v < VEC; ++v) as[(part * VEC + v) * LDA + r] = a_stage[i].v[v];
      } else {
        const int kk = c / Cfg::AT_CHUNKS_PER_ROW;
        const int part = c % Cfg::AT_CHUNKS_PER_ROW;
        *reinterpret_cast<Chunk16<T> *>(as + kk * LDA + part * VEC) = a_stage[i];
      }
    }
  };

  const unsigned k_tiles = size_k / BK;
  load_b_tma(0, 0);
  load_global(0);
  store_shared(0);
  __syncthreads();
  ptx::mbar_wait(bar0, 0);

  for (unsigned kt = 0; kt < k_tiles; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < k_tiles) {
      load_b_tma(buf ^ 1, (kt + 1) * BK);
      load_global((kt + 1) * BK);
    }

    const T *as = As + buf * BK * LDA;
    const T *bs = Bs + buf * BK * BN;
    const unsigned kbase = kt * BK;
#pragma unroll 1  // one pair of k per iteration: unrolled, some instantiations spill (see the top of the file)
    for (int kk = 0; kk < BK; kk += 2) {
      T af[2][8], bf[2][TN];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const Quad<T> a0 = *reinterpret_cast<const Quad<T> *>(as + (kk + u) * LDA + ty * 4);
        const Quad<T> a1 = *reinterpret_cast<const Quad<T> *>(as + (kk + u) * LDA + 64 + ty * 4);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          af[u][q] = a0.v[q];
          af[u][4 + q] = a1.v[q];
        }
#pragma unroll
        for (int h = 0; h < TN / 4; ++h) {
          const Quad<T> b = *reinterpret_cast<const Quad<T> *>(bs + (kk + u) * BN + h * 64 + tx * 4);
#pragma unroll
          for (int q = 0; q < 4; ++q) bf[u][h * 4 + q] = b.v[q];
        }
      }
      const unsigned k0 = kbase + kk;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
#pragma unroll
        for (int j = 0; j < TN; ++j) {
          witness_step<Map, Reduce>(acc[i][j], wit[i][j], af[0][i], bf[0][j], k0);
          witness_step<Map, Reduce>(acc[i][j], wit[i][j], af[1][i], bf[1][j], k0 + 1);
        }
      }
    }

    if (kt + 1 < k_tiles) store_shared(buf ^ 1);
    __syncthreads();
    if (kt + 1 < k_tiles) ptx::mbar_wait(bar0 + 8 * (buf ^ 1), ((kt + 1) >> 1) & 1u);
  }

  witness_epilogue<T, TN>(acc, wit, C, W, row0, col0, tx, ty, size_n, size_m);
}

// TMA-ring witness kernel: 4-byte types, A row-major; the SemiringRing geometry, stages handed over through full /
// empty mbarriers, no block-wide barrier in the main loop (see semiring_ring_kernel).
template <typename T, class Map, class Reduce>
__global__ void __launch_bounds__(256, 1)
semiring_witness_ring_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                             T *__restrict__ C, unsigned *__restrict__ W, unsigned size_n, unsigned size_k,
                             unsigned size_m, unsigned a_step, unsigned b_step) {
  static_assert(sizeof(T) == 4, "ring variant: 4-byte element types");
  using Cfg = SemiringRing;
  constexpr int BM = Cfg::BM, BN = Cfg::BN, BK = Cfg::BK, STAGES = Cfg::STAGES;
  C += size_t(blockIdx.z) * size_n * size_m;
  W += size_t(blockIdx.z) * size_n * size_m;
  const unsigned a_row0 = blockIdx.z * a_step * size_n, b_k0 = blockIdx.z * b_step * size_k;

  extern __shared__ unsigned char smem_raw[];
  const uint32_t smem0 = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t full0 = smem0 + STAGES * Cfg::STAGE_BYTES, empty0 = full0 + 8 * STAGES;

  const int tid = threadIdx.x, lane = tid % 32;
  const int tx = tid % 16;  // column quad index
  const int ty = tid / 16;  // row quad index
  const unsigned row0 = blockIdx.y * BM, col0 = blockIdx.x * BN;
  const unsigned k_tiles = size_k / BK;

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

  auto load_tile = [&](unsigned kt) {
    const int stage = kt % STAGES;
    if (kt >= STAGES) ptx::mbar_wait(empty0 + 8 * stage, ((kt / STAGES) - 1) & 1);
    const uint32_t as = smem0 + stage * Cfg::STAGE_BYTES, bs = as + Cfg::A_BYTES, bar = full0 + 8 * stage;
    ptx::mbar_arrive_expect_tx(bar, Cfg::STAGE_BYTES);
    ptx::tma_load_2d(as, &tmap_a, bar, int32_t(kt * BK), int32_t(a_row0 + row0), ptx::L2_EVICT_NORMAL);
    ptx::tma_load_2d(bs, &tmap_b, bar, int32_t(col0), int32_t(b_k0 + kt * BK), ptx::L2_EVICT_NORMAL);
  };
  if (tid == 0) {
    for (unsigned kt = 0; kt < unsigned(Cfg::AHEAD) && kt < k_tiles; ++kt) load_tile(kt);
  }

  T acc[8][8];
  unsigned wit[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      acc[i][j] = Reduce::identity();
      wit[i][j] = MM_WITNESS_NONE;
    }
  }

  const int r_lo = ty * 4, r_hi = 64 + ty * 4;

  for (unsigned kt = 0; kt < k_tiles; ++kt) {
    const int stage = kt % STAGES;
    if (tid == 0 && kt + Cfg::AHEAD < k_tiles) load_tile(kt + Cfg::AHEAD);
    ptx::mbar_wait(full0 + 8 * stage, (kt / STAGES) & 1);
    const unsigned char *as = smem_raw + (smem0 - ptx::smem_u32(smem_raw)) + stage * Cfg::STAGE_BYTES;
    const T *bs = reinterpret_cast<const T *>(as + Cfg::A_BYTES);
    const unsigned kbase = kt * BK;

#pragma unroll
    for (int c = 0; c < BK / 4; ++c) {  // four k per 16-byte chunk of an A row
      T a4[8][4];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int r = (i < 4 ? r_lo : r_hi) + (i % 4);
        const Quad<T> q = *reinterpret_cast<const Quad<T> *>(as + r * 64 + c * 16);
#pragma unroll
        for (int v = 0; v < 4; ++v) a4[i][v] = q.v[v];
      }
#pragma unroll
      for (int kp = 0; kp < 4; kp += 2) {
        const int kk = c * 4 + kp;
        T bf[2][8];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const Quad<T> b0 = *reinterpret_cast<const Quad<T> *>(bs + (kk + u) * BN + tx * 4);
          const Quad<T> b1 = *reinterpret_cast<const Quad<T> *>(bs + (kk + u) * BN + 64 + tx * 4);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            bf[u][q] = b0.v[q];
            bf[u][4 + q] = b1.v[q];
          }
        }
        const unsigned k0 = kbase + kk;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            witness_step<Map, Reduce>(acc[i][j], wit[i][j], a4[i][kp], bf[0][j], k0);
            witness_step<Map, Reduce>(acc[i][j], wit[i][j], a4[i][kp + 1], bf[1][j], k0 + 1);
          }
        }
      }
    }
    __syncwarp();
    if (lane == 0) ptx::mbar_arrive(empty0 + 8 * stage);  // this warp is done reading the stage
  }

  witness_epilogue<T, 8>(acc, wit, C, W, row0, col0, tx, ty, size_n, size_m);
}

// Host side.  Returns a cudaError_t value as int.
template <typename T, class Map, class Reduce>
int launch_semiring_witness_typed(const GemmArgs &g, unsigned *w, bool transposed_a, bool ring) {
  const GemmBatch &batch = g.batch;
  const unsigned n = g.n, k = g.k, m = g.m;
  CUtensorMap tmap_a, tmap_b;
  const uint64_t a_rows = uint64_t(batch.a_copies()) * n, b_rows = uint64_t(batch.b_copies()) * k;
  const unsigned a_step = batch.shared_a ? 0u : 1u, b_step = batch.shared_b ? 0u : 1u;
  if constexpr (sizeof(T) == 4) {
    if (ring && !transposed_a) {
      using Cfg = SemiringRing;
      auto kernel = semiring_witness_ring_kernel<T, Map, Reduce>;
      cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(Cfg::SMEM_BYTES));
      if (e != cudaSuccess) return static_cast<int>(e);
      if (encode_plain_2d(&tmap_a, g.a, sizeof(T), a_rows, k, Cfg::BM, Cfg::BK) != 0 ||
          encode_plain_2d(&tmap_b, g.b, sizeof(T), b_rows, m, Cfg::BK, Cfg::BN) != 0) {
        return static_cast<int>(cudaErrorInvalidValue);
      }
      dim3 grid((m + Cfg::BN - 1) / Cfg::BN, (n + Cfg::BM - 1) / Cfg::BM, batch.count);
      kernel<<<grid, Cfg::THREADS, Cfg::SMEM_BYTES, g.stream>>>(tmap_a, tmap_b, static_cast<T *>(g.c), w, n, k, m,
                                                                 a_step, b_step);
      return static_cast<int>(cudaGetLastError());
    }
  }
  using Cfg = WitnessTile<T>;
  if (encode_plain_2d(&tmap_b, g.b, sizeof(T), b_rows, m, Cfg::BK, Cfg::BN) != 0) {
    return static_cast<int>(cudaErrorInvalidValue);
  }
  dim3 grid((m + Cfg::BN - 1) / Cfg::BN, (n + Cfg::BM - 1) / Cfg::BM, batch.count);
  semiring_witness_tile_kernel<T, Map, Reduce><<<grid, Cfg::THREADS, Cfg::SMEM_BYTES, g.stream>>>(
      static_cast<const T *>(g.a), tmap_b, static_cast<T *>(g.c), w, n, k, m, transposed_a, a_step, b_step);
  return static_cast<int>(cudaGetLastError());
}

// One translation unit per (data type, map operator) instantiates the Min / Max reduces, plus the FMNMX pair for
// float (semiring_witness_inst.cu compiled with -DMM_INST_T=<type> -DMM_INST_MAP=<MM_OP_*>).
template <typename T, int MAP_OP>
int launch_semiring_witness_for(int reduce_op, const GemmArgs &g, unsigned *w, bool ta, bool ring);

#define MM_WITNESS_CASE(REDOP)                                                                      \
  if (reduce_op == REDOP)                                                                           \
    return launch_semiring_witness_typed<T, typename OpSelect<T, MAP_OP>::type,                     \
                                         typename OpSelect<T, REDOP>::type>(g, w, ta, ring);

#define MM_INSTANTIATE_SEMIRING_WITNESS(TYPE, MAPOP)                                                \
  template <>                                                                                       \
  int launch_semiring_witness_for<TYPE, MAPOP>(int reduce_op, const GemmArgs &g, unsigned *w, bool ta, \
                                               bool ring) {                                        \
    using T = TYPE;                                                                                 \
    constexpr int MAP_OP = MAPOP;                                                                   \
    MM_WITNESS_CASE(MM_OP_MIN)                                                                      \
    MM_WITNESS_CASE(MM_OP_MAX)                                                                      \
    if constexpr (std::is_same<T, float>::value) {                                                  \
      MM_WITNESS_CASE(MM_OP_MIN_FAST)                                                               \
      MM_WITNESS_CASE(MM_OP_MAX_FAST)                                                               \
    }                                                                                               \
    return -1;                                                                                      \
  }

}  // namespace mm
