// CUDA-core semiring tile kernel:  C[N x M] = A[N x K] (x) B[K x M]  for ANY (Map, Reduce, T).
//
// sm_90a counterpart of the reference's ProcessingElement chain (kernel/Compute.cpp:11-231) fed by
// ReadA/TransposeA/ReadB/FeedB and drained by WriteC (kernel/Memory.cpp:58-438), for the
// configurations that are not a dense (Multiply, Add) contraction on a tensor-core type — and,
// under MM_FLAG_EXACT, for those too.  Like the reference it computes an outer product per k into
// an on-chip C tile that is written once; unlike the reference's literal-0 seed
// (kernel/Compute.cpp:116-118, which breaks Min — SURVEY.md section 5 trap 1) the accumulators
// start from OperatorReduce::identity(), the result definition of Naive<> (include/Utility.h:29).
//
// Exactness: every C element is reduced by ONE thread, sequentially over k = 0..K-1, with one
// rounding per Map and per Reduce (semiring.cuh), so the output is bit-identical to Naive<>.
//
// Tiling: CTA tile BM x BN = 128 x 128, k-step BK = 64 bytes of K (the reference's memory word,
// so K % BK == 0 is implied by the reference's own shape rule), 256 threads, 8 x 8 accumulators
// per thread laid out as 2 x 2 quads of 4 so that shared-memory fragment reads are 16-byte
// conflict-free and global C stores are row-contiguous.  A is transposed on the way into shared
// memory (the role of TransposeA, kernel/Memory.cpp:130-181) through registers, with the next
// tile's global loads in flight during the current tile's compute; the B tile (BK rows x 128
// columns, natural orientation — the role of ReadB/FeedB) is staged by TMA
// (cp.async.bulk.tensor + mbarrier complete_tx), the same mechanism the tensor-core path uses.
// No warp-shuffle reduction is needed (or wanted): K is never split across lanes, which is what
// keeps the reduction order — and therefore every rounding — identical to Naive<>.
//
// Batch: blockIdx.z = problem.  B's map holds the problems stacked along K (a tile never crosses a
// problem: K % BK == 0); A and C take per-problem pointer offsets.  a_step / b_step: 1 = packed
// operands, 0 = every problem reads problem 0's.
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <type_traits>

#include "common.cuh"
#include "ptx_sm90.cuh"
#include "semiring.cuh"
#include "tma_host.cuh"

namespace mm {

template <typename T>
struct alignas((sizeof(T) * 4 <= 16) ? sizeof(T) * 4 : 16) Quad {
  T v[4];
};

template <typename T>
struct alignas(16) Chunk16 {  // one 16-byte global load
  T v[16 / sizeof(T)];
};

template <typename T>
struct SemiringTile {
  static constexpr int BM = 128;
  static constexpr int BN = 128;
  static constexpr int BK = 64 / sizeof(T);   // elements of K per step (64 bytes)
  static constexpr int VEC = 16 / sizeof(T);  // elements per 16-byte chunk
  static constexpr int THREADS = 256;
  // 128 rows x 64 B of A and BK rows x 128 cols of B are both 512 16-byte chunks.
  static constexpr int CHUNKS = 512;
  static constexpr int CHUNKS_PER_THREAD = CHUNKS / THREADS;  // 2
  static constexpr int A_CHUNKS_PER_ROW = BK / VEC;           // 4
  static constexpr int B_CHUNKS_PER_ROW = BN / VEC;
  static constexpr int PAD = 4;                               // elements; keeps 16 B alignment for T >= 4 B
  static constexpr int LDA = BM + ((sizeof(T) >= 4) ? PAD : 16 / sizeof(T));
  static constexpr int LDB = BN;
  static constexpr size_t A_BYTES = (2 * size_t(BK) * LDA * sizeof(T) + 127) / 128 * 128;  // keeps Bs 128-B aligned
  static constexpr size_t B_TILE_BYTES = size_t(BK) * LDB * sizeof(T);                     // one TMA box
  static constexpr size_t SMEM_BYTES = A_BYTES + 2 * B_TILE_BYTES + 16 /* two mbarriers */;
};

// half with a Sum / Product Map AND Reduce keeps its accumulators as __half2 pairs of adjacent columns (HADD2 / HMUL2).
template <typename T, class Map, class Reduce>
struct SemiringHalf2 {
  static constexpr bool value = std::is_same<T, __half>::value && PackedOpH<Map>::value && PackedOpH<Reduce>::value;
};
// bfloat16 likewise, as __nv_bfloat162 pairs (HADD2.BF16 / HMUL2.BF16).
template <typename T, class Map, class Reduce>
struct SemiringBf162 {
  static constexpr bool value =
      std::is_same<T, __nv_bfloat16>::value && PackedOpB<Map>::value && PackedOpB<Reduce>::value;
};

// ACC: C = Reduce(C_old, result), applied in the epilogue to the old C at the addresses about to be stored
// (semiring_accumulate_tile_kernel); nothing else differs.
template <typename T, class Map, class Reduce, bool ACC>
__device__ __forceinline__ void semiring_tile_body(const T *__restrict__ A, const CUtensorMap &tmap_b,
                                                   T *__restrict__ C, unsigned size_n, unsigned size_k,
                                                   unsigned size_m, bool TRANSPOSED_A, unsigned a_step,
                                                   unsigned b_step) {
  using Cfg = SemiringTile<T>;
  constexpr int BM = Cfg::BM, BN = Cfg::BN, BK = Cfg::BK, VEC = Cfg::VEC;
  constexpr int LDA = Cfg::LDA, LDB = Cfg::LDB;
  A += size_t(blockIdx.z * a_step) * size_n * size_k;
  C += size_t(blockIdx.z) * size_n * size_m;
  const unsigned b_k0 = blockIdx.z * b_step * size_k;  // first row of this problem's B in the map

  extern __shared__ __align__(128) unsigned char smem_raw[];
  T *As = reinterpret_cast<T *>(smem_raw);                          // [2][BK][LDA]  (k-major: A transposed)
  T *Bs = reinterpret_cast<T *>(smem_raw + Cfg::A_BYTES);           // [2][BK][LDB]  (TMA destination)
  const uint32_t bar0 = ptx::smem_u32(smem_raw + Cfg::A_BYTES + 2 * Cfg::B_TILE_BYTES);  // full[0], full[1]

  const int tid = threadIdx.x;
  const int tx = tid % 16;  // column quad index
  const int ty = tid / 16;  // row quad index
  const size_t row0 = size_t(blockIdx.y) * BM;
  const size_t col0 = size_t(blockIdx.x) * BN;

  constexpr bool kBf162 = SemiringBf162<T, Map, Reduce>::value;
  constexpr bool kHalf2 = SemiringHalf2<T, Map, Reduce>::value || kBf162;  // a packed pair path
  using P2 = Packed2<T>;
  using T2 = typename P2::type;
  using MapOp2 = typename std::conditional<kBf162, PackedOpB<Map>, PackedOpH<Map>>::type;
  using ReduceOp2 = typename std::conditional<kBf162, PackedOpB<Reduce>, PackedOpH<Reduce>>::type;
  T acc[8][8];
  T2 acc2[8][4];  // kHalf2 only: columns (2p, 2p + 1) of row i
#pragma unroll
  for (int i = 0; i < 8; ++i) {
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = Reduce::identity();
    if constexpr (kHalf2) {
#pragma unroll
      for (int p = 0; p < 4; ++p) acc2[i][p] = P2::bcast(Reduce::identity());
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
  // B tile kt -> Bs[buf]: one elected thread arms the barrier with the byte count and issues the TMA
  auto load_b_tma = [&](int buf, unsigned k0) {
    if (tid == 0) {
      ptx::mbar_arrive_expect_tx(bar0 + 8 * buf, uint32_t(Cfg::B_TILE_BYTES));
      ptx::tma_load_2d(ptx::smem_u32(Bs + buf * BK * LDB), &tmap_b, bar0 + 8 * buf, int32_t(col0), int32_t(b_k0 + k0),
                       ptx::L2_EVICT_NORMAL);
    }
  };

  auto load_global = [&](unsigned k0) {
#pragma unroll
    for (int i = 0; i < Cfg::CHUNKS_PER_THREAD; ++i) {
      const int c = tid + i * Cfg::THREADS;
      if (!TRANSPOSED_A) {
        // A row-major N x K: chunk = (row, 16-byte part of the 64-byte k-slab)
        const int r = c / Cfg::A_CHUNKS_PER_ROW;
        const int part = c % Cfg::A_CHUNKS_PER_ROW;
        size_t row = row0 + r;
        if (row >= size_n) row = size_n - 1;  // clamp: rows past N are computed but never stored
        a_stage[i] = *reinterpret_cast<const Chunk16<T> *>(A + row * size_k + k0 + part * VEC);
      } else {
        // A stored K x N: element-wise (N need not be a multiple of the vector width)
        const int kk = c / Cfg::B_CHUNKS_PER_ROW;
        const int part = c % Cfg::B_CHUNKS_PER_ROW;
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
        const int kk = c / Cfg::B_CHUNKS_PER_ROW;
        const int part = c % Cfg::B_CHUNKS_PER_ROW;
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
      // buffer buf^1 was last read in iteration kt-1, which ended with a __syncthreads()
      load_b_tma(buf ^ 1, (kt + 1) * BK);
      load_global((kt + 1) * BK);
    }

    const T *as = As + buf * BK * LDA;
    const T *bs = Bs + buf * BK * LDB;
#pragma unroll
    for (int kk = 0; kk < BK; kk += 2) {
      // two consecutive k per step, reduced in order inside ONE expression
      //   acc = Reduce(Reduce(acc, Map(a_k, b_k)), Map(a_k+1, b_k+1))
      // so that a 3-input hardware reduction can be selected where the target has one; the
      // evaluation order, and therefore every rounding, is the sequential order of Naive<>.
      T af[2][8], bf[2][8];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const Quad<T> a0 = *reinterpret_cast<const Quad<T> *>(as + (kk + u) * LDA + ty * 4);
        const Quad<T> a1 = *reinterpret_cast<const Quad<T> *>(as + (kk + u) * LDA + 64 + ty * 4);
        const Quad<T> b0 = *reinterpret_cast<const Quad<T> *>(bs + (kk + u) * LDB + tx * 4);
        const Quad<T> b1 = *reinterpret_cast<const Quad<T> *>(bs + (kk + u) * LDB + 64 + tx * 4);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          af[u][q] = a0.v[q];
          af[u][4 + q] = a1.v[q];
          bf[u][q] = b0.v[q];
          bf[u][4 + q] = b1.v[q];
        }
      }
      if constexpr (kHalf2) {
        // half / bfloat16, Map and Reduce in {Sum, Product}: two adjacent columns per HMUL2 / HADD2 (A element
        // broadcast by the instruction's half selector), one rounding per Map and per Reduce per element, in
        // Naive<>'s order
        T2 bp[2][4];
#pragma unroll
        for (int u = 0; u < 2; ++u)
#pragma unroll
          for (int p = 0; p < 4; ++p) bp[u][p] = P2::pair(bf[u][2 * p], bf[u][2 * p + 1]);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const T2 a0 = P2::bcast(af[0][i]), a1 = P2::bcast(af[1][i]);
#pragma unroll
          for (int p = 0; p < 4; ++p) {
            const T2 t0 = MapOp2::Apply2(a0, bp[0][p]), t1 = MapOp2::Apply2(a1, bp[1][p]);
            acc2[i][p] = ReduceOp2::Apply2(ReduceOp2::Apply2(acc2[i][p], t0), t1);
          }
        }
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            acc[i][j] = Reduce::Apply(Reduce::Apply(acc[i][j], Map::Apply(af[0][i], bf[0][j])),
                                      Map::Apply(af[1][i], bf[1][j]));
          }
        }
      }
    }

    if (kt + 1 < k_tiles) store_shared(buf ^ 1);
    __syncthreads();
    // tile kt+1 of B: phase parity of barrier (buf^1) = number of earlier uses of that buffer, mod 2
    if (kt + 1 < k_tiles) ptx::mbar_wait(bar0 + 8 * (buf ^ 1), ((kt + 1) >> 1) & 1u);
  }

  // Write the C tile once, masked to n < N, m < M (the role of WriteC, kernel/Memory.cpp:361-392).
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const size_t row = row0 + (i / 4) * 64 + ty * 4 + (i % 4);
    if (row >= size_n) continue;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const size_t col = col0 + h * 64 + tx * 4;
      if (col + 4 <= size_m) {
        Quad<T> out;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          if constexpr (kHalf2) {
            out.v[q] = (q % 2 == 0) ? P2::lo(acc2[i][h * 2 + q / 2]) : P2::hi(acc2[i][h * 2 + q / 2]);
          } else {
            out.v[q] = acc[i][h * 4 + q];
          }
        }
        if constexpr (ACC) {
          const Quad<T> old = *reinterpret_cast<const Quad<T> *>(C + row * size_m + col);
#pragma unroll
          for (int p = 0; p < 4; p += 2) {
            if constexpr (kHalf2) {
              const T2 r = ReduceOp2::Apply2(P2::pair(old.v[p], old.v[p + 1]), P2::pair(out.v[p], out.v[p + 1]));
              out.v[p] = P2::lo(r);
              out.v[p + 1] = P2::hi(r);
            } else {
              out.v[p] = Reduce::Apply(old.v[p], out.v[p]);
              out.v[p + 1] = Reduce::Apply(old.v[p + 1], out.v[p + 1]);
            }
          }
        }
        *reinterpret_cast<Quad<T> *>(C + row * size_m + col) = out;
      }
    }
  }
}

// 2 CTAs (16 warps) per SM for 4-byte element types and packed half / bfloat16: 64 accumulators + two k-steps of fragments fit
// in 128 registers without spilling.  8-byte types need the full 255-register budget, and unpacked 1- and
// 2-byte types (one 32-bit register per element) spill at 128: those run 1 CTA per SM.
template <typename T, class Map, class Reduce>
__global__ void __launch_bounds__(256, (sizeof(T) == 4 || SemiringHalf2<T, Map, Reduce>::value ||
                                       SemiringBf162<T, Map, Reduce>::value) ? 2 : 1)
semiring_tile_kernel(const T *__restrict__ A, const __grid_constant__ CUtensorMap tmap_b, T *__restrict__ C,
                     unsigned size_n, unsigned size_k, unsigned size_m,
                     bool TRANSPOSED_A, unsigned a_step, unsigned b_step) {
  semiring_tile_body<T, Map, Reduce, false>(A, tmap_b, C, size_n, size_k, size_m, TRANSPOSED_A, a_step, b_step);
}

// C <- Reduce(C_old, A (x) B) (mm_kernel_enqueue_accumulate); instantiated by semiring_accumulate_inst.cu only.
template <typename T, class Map, class Reduce>
__global__ void __launch_bounds__(256, (sizeof(T) == 4 || SemiringHalf2<T, Map, Reduce>::value ||
                                       SemiringBf162<T, Map, Reduce>::value) ? 2 : 1)
semiring_accumulate_tile_kernel(const T *__restrict__ A, const __grid_constant__ CUtensorMap tmap_b,
                                T *__restrict__ C, unsigned size_n, unsigned size_k, unsigned size_m,
                                bool TRANSPOSED_A, unsigned a_step, unsigned b_step) {
  semiring_tile_body<T, Map, Reduce, true>(A, tmap_b, C, size_n, size_k, size_m, TRANSPOSED_A, a_step, b_step);
}

}  // namespace mm

#include "semiring_ring_kernel.cuh"  // uses Quad<T> from above

namespace mm {

// Only the kernels a translation unit launches are instantiated there.
template <typename T, class Map, class Reduce, bool ACC>
constexpr auto semiring_tile_kernel_ptr() {
  if constexpr (ACC) return semiring_accumulate_tile_kernel<T, Map, Reduce>;
  else return semiring_tile_kernel<T, Map, Reduce>;
}

// ACC: the accumulate kernels, with the same choice between the ring and the tile kernel.
template <typename T, class Map, class Reduce, bool ACC = false>
int launch_semiring_typed(const void *a, const void *b, void *c, unsigned n, unsigned k, unsigned m,
                          bool transposed_a, bool ring, const GemmBatch &batch, cudaStream_t stream) {
  using Cfg = SemiringTile<T>;
  if constexpr (sizeof(T) == 4) {
    // 4-byte types with A stored row-major take the ring variant (both tiles by TMA, no block-wide barrier:
    // 41.7 vs 39.9 TOp/s for float (Add, Min) at 8192^3); the tuning knob MM_TUNE_SEMIRING_RING = 0 keeps this kernel
    if (ring && !transposed_a && (a == nullptr || reinterpret_cast<uintptr_t>(a) % 16 == 0)) {
      return launch_semiring_ring<T, Map, Reduce, ACC>(a, b, c, n, k, m, batch.count, batch.shared_a, batch.shared_b,
                                                       stream);
    }
  }
  if (a == nullptr) {  // dry run: only make sure the kernel is loaded
    cudaFuncAttributes attr;
    return static_cast<int>(cudaFuncGetAttributes(&attr, semiring_tile_kernel_ptr<T, Map, Reduce, ACC>()));
  }
  dim3 grid((m + Cfg::BN - 1) / Cfg::BN, (n + Cfg::BM - 1) / Cfg::BM, batch.count);
  dim3 block(Cfg::THREADS);
  const T *pa = static_cast<const T *>(a);
  T *pc = static_cast<T *>(c);
  // B row-major K x M (the problems of a batch stacked along K), box = BK rows x 128 columns
  CUtensorMap tmap_b;
  const uint64_t b_rows = uint64_t(batch.shared_b ? 1 : batch.count) * k;
  if (encode_plain_2d(&tmap_b, b, sizeof(T), b_rows, m, Cfg::BK, Cfg::BN) != 0) {
    return static_cast<int>(cudaErrorInvalidValue);
  }
  semiring_tile_kernel_ptr<T, Map, Reduce, ACC>()<<<grid, block, Cfg::SMEM_BYTES, stream>>>(
      pa, tmap_b, pc, n, k, m, transposed_a, batch.shared_a ? 0u : 1u, batch.shared_b ? 0u : 1u);
  return static_cast<int>(cudaGetLastError());
}

// One translation unit per (data type, map operator) instantiates the five reduce operators
// (semiring_inst.cu compiled with -DMM_INST_T=<type> -DMM_INST_MAP=<MM_OP_*>); 30 small units
// build in parallel.
template <typename T, int MAP_OP>
int launch_semiring_for(int reduce_op, const void *a, const void *b, void *c, unsigned n, unsigned k,
                        unsigned m, bool ta, bool ring, const GemmBatch &batch, cudaStream_t stream);

// The same for the accumulate kernels (semiring_accumulate_inst.cu).
template <typename T, int MAP_OP>
int launch_semiring_accumulate_for(int reduce_op, const void *a, const void *b, void *c, unsigned n, unsigned k,
                                   unsigned m, bool ta, bool ring, const GemmBatch &batch, cudaStream_t stream);

#define MM_SEMIRING_CASE(REDOP)                                                                    \
  if (reduce_op == REDOP)                                                                          \
    return launch_semiring_typed<T, typename OpSelect<T, MAP_OP>::type,                            \
                                 typename OpSelect<T, REDOP>::type, ACC>(a, b, c, n, k, m, ta, ring, batch, stream);

#define MM_INSTANTIATE_SEMIRING_FN(FN, ACCV, TYPE, MAPOP)                                          \
  template <>                                                                                      \
  int FN<TYPE, MAPOP>(int reduce_op, const void *a, const void *b, void *c,                        \
                      unsigned n, unsigned k, unsigned m, bool ta, bool ring,                      \
                      const GemmBatch &batch, cudaStream_t stream) {                               \
    using T = TYPE;                                                                                \
    constexpr int MAP_OP = MAPOP;                                                                  \
    constexpr bool ACC = ACCV;                                                                     \
    MM_SEMIRING_CASE(MM_OP_MULTIPLY)                                                               \
    MM_SEMIRING_CASE(MM_OP_ADD)                                                                    \
    MM_SEMIRING_CASE(MM_OP_MIN)                                                                    \
    MM_SEMIRING_CASE(MM_OP_MAX)                                                                    \
    MM_SEMIRING_CASE(MM_OP_AND)                                                                    \
    if constexpr (std::is_same<T, float>::value) {                                                 \
      MM_SEMIRING_CASE(MM_OP_MIN_FAST)                                                             \
      MM_SEMIRING_CASE(MM_OP_MAX_FAST)                                                             \
    }                                                                                              \
    return -1;                                                                                     \
  }
#define MM_INSTANTIATE_SEMIRING(TYPE, MAPOP) MM_INSTANTIATE_SEMIRING_FN(launch_semiring_for, false, TYPE, MAPOP)
#define MM_INSTANTIATE_SEMIRING_ACCUMULATE(TYPE, MAPOP) \
  MM_INSTANTIATE_SEMIRING_FN(launch_semiring_accumulate_for, true, TYPE, MAPOP)

}  // namespace mm
