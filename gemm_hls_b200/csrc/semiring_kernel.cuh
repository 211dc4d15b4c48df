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
//
// One main loop per scheme.  semiring_tile_body (here) and semiring_ring_body (semiring_ring_kernel.cuh) are the only
// main loops of the register-staged and the TMA-ring scheme; every kernel of the family (plain, accumulate, witness,
// closure phase 3) is a thin __global__ wrapper that computes where its operands start and passes a variant: a type
// that supplies only what differs between the callers (SemiringVariant below).
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

// TN: columns of C per thread (8, or 4 for the witness kernel's 128 x 64 CTA tile).
template <typename T, int TN = 8>
struct SemiringTile {
  static constexpr int BM = 128;
  static constexpr int BN = 16 * TN;
  static constexpr int BK = 64 / sizeof(T);   // elements of K per step (64 bytes)
  static constexpr int VEC = 16 / sizeof(T);  // elements per 16-byte chunk
  static constexpr int THREADS = 256;
  // 128 rows x 64 B of A is 512 16-byte chunks.
  static constexpr int CHUNKS = 512;
  static constexpr int CHUNKS_PER_THREAD = CHUNKS / THREADS;  // 2
  static constexpr int A_CHUNKS_PER_ROW = BK / VEC;           // row-major A: per row of A (4)
  static constexpr int AT_CHUNKS_PER_ROW = BM / VEC;          // A stored K x N: per k
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

// The term Map(a, b) as apply(prep(a), prep(b)); prep runs once per operand as it leaves shared memory.
template <class Map>
struct MapTerm {
  template <typename T>
  static __device__ __forceinline__ T prep(T x) { return x; }
  template <typename T>
  static __device__ __forceinline__ T apply(T a, T b) { return Map::Apply(a, b); }
};

// What a caller of the main loops supplies, with the product's defaults.  A variant defines
//   Term                   the term, as above;
//   State                  a register the step keeps beside each accumulator (the witness), or NoState;
//   TN, kRolledK, kLateA   the tile body's geometry: columns per thread, one pair of k per loop iteration instead of
//                          the whole k-tile unrolled, and the next A tile loaded after the compute instead of before;
//   kMaxK                  a bound on the rows of B the loop covers (the closure's block width);
//   C, size_n, size_m      problem 0's C and every problem's extents: problem z's C starts z * size_n * size_m later;
//   seed(acc, state, C, row0, col0, tx, ty)     the accumulators' start (default: the reduce's identity);
//   kSeedC                 the tile body seeds the accumulators itself with the C tile, the reduce's identity outside
//                          it, instead of calling seed;
//   step(acc, state, a0, b0, a1, b1, k)         the accumulator after the pair k, k + 1, k counted within the problem
//                                               (default: the plain pair below);
//   kAccumulate            the body's epilogue stores Reduce(C_old, result), applied to the old C at the addresses
//                          about to be stored (mm_kernel_enqueue_accumulate), instead of the result;
//   kFinish, finish(acc, state, row0, col0, tx, ty)   an epilogue of the variant's own instead of the body's.
// Thread (tx, ty) owns rows (i / 4) * 64 + ty * 4 + i % 4 (i < 8) and columns (j / 4) * 64 + tx * 4 + j % 4 (j < TN) of
// the CTA tile at (row0, col0); C is the problem's.  The bodies keep their own epilogue and C-tile seed, the batch
// offsets, the K bound and the step's assignment inline, and the step takes its operands by reference: written
// otherwise, the product kernels' machine code changes and the closure kernels take more registers.
struct NoState {};

template <typename T_, class Map_, class Reduce_, bool ACC = false, class Term_ = MapTerm<Map_>>
struct SemiringVariant {
  using T = T_;
  using Map = Map_;
  using Reduce = Reduce_;
  using Term = Term_;
  using State = NoState;
  static constexpr int TN = 8;
  static constexpr bool kRolledK = false, kLateA = false, kSeedC = false, kAccumulate = ACC, kFinish = false;
  static constexpr unsigned kMaxK = ~0u;
  T *C;
  unsigned size_n, size_m;

  template <typename I>
  __device__ __forceinline__ void seed(T (&acc)[8][TN], State (&)[8][TN], const T *, I, I, int, int) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int j = 0; j < TN; ++j) acc[i][j] = Reduce::identity();
    }
  }
  // two consecutive k per step, reduced in order inside ONE expression
  //   acc = Reduce(Reduce(acc, Map(a_k, b_k)), Map(a_k+1, b_k+1))
  // so that a 3-input hardware reduction can be selected where the target has one; the
  // evaluation order, and therefore every rounding, is the sequential order of Naive<>.
  __device__ __forceinline__ T step(const T &acc, State &, const T &a0, const T &b0, const T &a1, const T &b1,
                                    unsigned) {
    return Reduce::Apply(Reduce::Apply(acc, Term::apply(a0, b0)), Term::apply(a1, b1));
  }
};

// The register-staged main loop.  Problem blockIdx.z reads A at A + blockIdx.z * a_step * size_n * lda (row-major,
// row pitch lda; A stored K x N has row pitch size_n) and B from row blockIdx.z * b_step * b_rows + b_k0 of the map.
// A goes through registers and is transposed into shared memory; B arrives by TMA.  The loop covers B's rows from b_k0
// to the end of the problem (b_rows), at most V::kMaxK of them: a multiple of BK.
template <class V>
__device__ __forceinline__ void semiring_tile_body(V &&v, const typename V::T *__restrict__ A, unsigned a_step,
                                                   unsigned lda, bool TRANSPOSED_A, const CUtensorMap &tmap_b,
                                                   unsigned b_step, unsigned b_rows, unsigned b_k0) {
  using T = typename V::T;
  using Map = typename V::Map;
  using Reduce = typename V::Reduce;
  using Term = typename V::Term;
  constexpr int TN = V::TN;
  using Cfg = SemiringTile<T, TN>;
  constexpr int BM = Cfg::BM, BN = Cfg::BN, BK = Cfg::BK, VEC = Cfg::VEC;
  constexpr int LDA = Cfg::LDA, LDB = Cfg::LDB;
  const unsigned size_n = v.size_n, size_m = v.size_m;
  A += size_t(blockIdx.z * a_step) * size_n * lda;
  T *C = v.C + size_t(blockIdx.z) * size_n * size_m;
  const unsigned b_row0 = blockIdx.z * b_step * b_rows + b_k0;  // first row of this problem's B in the map

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
  // the packed pair path keeps its own accumulators, seed and step: the product's variant only
  static_assert(!kHalf2 || std::is_same<V, SemiringVariant<T, Map, Reduce, V::kAccumulate>>::value,
                "the packed pair path serves the product's variant only");
  using P2 = Packed2<T>;
  using T2 = typename P2::type;
  using MapOp2 = typename std::conditional<kBf162, PackedOpB<Map>, PackedOpH<Map>>::type;
  using ReduceOp2 = typename std::conditional<kBf162, PackedOpB<Reduce>, PackedOpH<Reduce>>::type;
  T acc[8][TN];
  typename V::State state[8][TN];
  T2 acc2[8][4];  // kHalf2 only: columns (2p, 2p + 1) of row i
  if constexpr (V::kSeedC) {
    // the C tile, masked to n < N, m < M, the reduce's identity outside it (inline, as the epilogue)
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const size_t row = row0 + (i / 4) * 64 + ty * 4 + (i % 4);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const size_t col = col0 + h * 64 + tx * 4;
        Quad<T> old;
        if (row < size_n && col + 4 <= size_m) {
          old = *reinterpret_cast<const Quad<T> *>(C + row * size_m + col);
        } else {
#pragma unroll
          for (int q = 0; q < 4; ++q) old.v[q] = Reduce::identity();
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[i][h * 4 + q] = old.v[q];
      }
    }
  } else {
    v.seed(acc, state, C, row0, col0, tx, ty);
  }
  if constexpr (kHalf2) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
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
      ptx::tma_load_2d(ptx::smem_u32(Bs + buf * BK * LDB), &tmap_b, bar0 + 8 * buf, int32_t(col0), int32_t(b_row0 + k0),
                       ptx::L2_EVICT_NORMAL);
    }
  };

  auto load_global = [&](unsigned k0) {
#pragma unroll
    for (int i = 0; i < Cfg::CHUNKS_PER_THREAD; ++i) {
      const int c = tid + i * Cfg::THREADS;
      if (!TRANSPOSED_A) {
        // A row-major: chunk = (row, 16-byte part of the 64-byte k-slab)
        const int r = c / Cfg::A_CHUNKS_PER_ROW;
        const int part = c % Cfg::A_CHUNKS_PER_ROW;
        size_t row = row0 + r;
        if (row >= size_n) row = size_n - 1;  // clamp: rows past N are computed but never stored
        a_stage[i] = *reinterpret_cast<const Chunk16<T> *>(A + row * lda + k0 + part * VEC);
      } else {
        // A stored K x N: element-wise (N need not be a multiple of the vector width)
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

  const unsigned k_tiles = min(b_rows - b_k0, V::kMaxK) / BK;
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
      if (!V::kLateA) load_global((kt + 1) * BK);
    }

    const T *as = As + buf * BK * LDA;
    const T *bs = Bs + buf * BK * LDB;
    constexpr int KK_UNROLL = V::kRolledK ? 1 : BK / 2;
#pragma unroll KK_UNROLL
    for (int kk = 0; kk < BK; kk += 2) {
      T af[2][8], bf[2][TN];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const Quad<T> a0 = *reinterpret_cast<const Quad<T> *>(as + (kk + u) * LDA + ty * 4);
        const Quad<T> a1 = *reinterpret_cast<const Quad<T> *>(as + (kk + u) * LDA + 64 + ty * 4);
        const Quad<T> b0 = *reinterpret_cast<const Quad<T> *>(bs + (kk + u) * LDB + tx * 4);
        // TN = 4: one quad of B, b1 = b0
        const Quad<T> b1 = *reinterpret_cast<const Quad<T> *>(bs + (kk + u) * LDB + (TN - 4) * 16 + tx * 4);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          af[u][q] = Term::prep(a0.v[q]);
          af[u][4 + q] = Term::prep(a1.v[q]);
          bf[u][q] = Term::prep(b0.v[q]);
          if constexpr (TN == 8) bf[u][4 + q] = Term::prep(b1.v[q]);
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
          for (int j = 0; j < TN; ++j) {
            acc[i][j] = v.step(acc[i][j], state[i][j], af[0][i], bf[0][j], af[1][i], bf[1][j], kt * BK + kk);
          }
        }
      }
    }

    if (kt + 1 < k_tiles) {
      if (V::kLateA) load_global((kt + 1) * BK);
      store_shared(buf ^ 1);
    }
    __syncthreads();
    // tile kt+1 of B: phase parity of barrier (buf^1) = number of earlier uses of that buffer, mod 2
    if (kt + 1 < k_tiles) ptx::mbar_wait(bar0 + 8 * (buf ^ 1), ((kt + 1) >> 1) & 1u);
  }

  if constexpr (V::kFinish) {
    v.finish(acc, state, row0, col0, tx, ty);
  } else {
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
          if constexpr (V::kAccumulate) {
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
}

// The product kernels: problem z reads the A of problem z * a_step and the B of problem z * b_step (a step of 0: every
// problem reads problem 0's).
template <typename T, class Map, class Reduce, bool ACC>
__device__ __forceinline__ void semiring_tile_product(const T *__restrict__ A, const CUtensorMap &tmap_b,
                                                      T *__restrict__ C, unsigned size_n, unsigned size_k,
                                                      unsigned size_m, bool TRANSPOSED_A, unsigned a_step,
                                                      unsigned b_step) {
  semiring_tile_body(SemiringVariant<T, Map, Reduce, ACC>{C, size_n, size_m}, A, a_step, size_k, TRANSPOSED_A, tmap_b,
                     b_step, size_k, 0u);
}

// 2 CTAs (16 warps) per SM for 4-byte element types and packed half / bfloat16: 64 accumulators + two k-steps of
// fragments fit in 128 registers without spilling.  8-byte types need the full 255-register budget, and unpacked 1- and
// 2-byte types (one 32-bit register per element) spill at 128: those run 1 CTA per SM.
template <typename T, class Map, class Reduce>
__global__ void __launch_bounds__(256, (sizeof(T) == 4 || SemiringHalf2<T, Map, Reduce>::value ||
                                       SemiringBf162<T, Map, Reduce>::value) ? 2 : 1)
semiring_tile_kernel(const T *__restrict__ A, const __grid_constant__ CUtensorMap tmap_b, T *__restrict__ C,
                     unsigned size_n, unsigned size_k, unsigned size_m,
                     bool TRANSPOSED_A, unsigned a_step, unsigned b_step) {
  semiring_tile_product<T, Map, Reduce, false>(A, tmap_b, C, size_n, size_k, size_m, TRANSPOSED_A, a_step, b_step);
}

// C <- Reduce(C_old, A (x) B) (mm_kernel_enqueue_accumulate); instantiated by semiring_accumulate_inst.cu only.
template <typename T, class Map, class Reduce>
__global__ void __launch_bounds__(256, (sizeof(T) == 4 || SemiringHalf2<T, Map, Reduce>::value ||
                                       SemiringBf162<T, Map, Reduce>::value) ? 2 : 1)
semiring_accumulate_tile_kernel(const T *__restrict__ A, const __grid_constant__ CUtensorMap tmap_b,
                                T *__restrict__ C, unsigned size_n, unsigned size_k, unsigned size_m,
                                bool TRANSPOSED_A, unsigned a_step, unsigned b_step) {
  semiring_tile_product<T, Map, Reduce, true>(A, tmap_b, C, size_n, size_k, size_m, TRANSPOSED_A, a_step, b_step);
}

}  // namespace mm

#include "semiring_ring_kernel.cuh"  // uses Quad<T> and the variants from above

namespace mm {

// ---- host side ----------------------------------------------------------------------------------------------------

// The ring kernel serves 4-byte types whose A is row-major and 16-byte aligned, unless the tuning knob
// MM_TUNE_SEMIRING_RING = 0 keeps the tile kernel (41.7 vs 39.9 TOp/s for float (Add, Min) at 8192^3); the
// register-staged tile kernel serves the rest.
template <typename T>
bool semiring_takes_ring(const void *a, bool transposed_a, bool ring) {
  return sizeof(T) == 4 && ring && !transposed_a && reinterpret_cast<uintptr_t>(a) % 16 == 0;
}

// Loads `kernel` with `smem` bytes of dynamic shared memory, encodes the tensor maps of its main loop over row-major
// operands whose problems are stacked along the rows, and runs launch(grid, tmap_a, tmap_b): A (a_rows x a_cols) in the
// ring's BM x BK boxes, the ring only (tmap_a stays unset for the tile kernel); B (b_rows x b_cols) in BK x BN boxes.
// The grid covers `rows` x `cols` of C per problem, `batch` problems.  Null A: a dry run that only loads the kernel.
// Returns a cudaError_t value as int.
template <typename T, int BN, class Kernel, class Launch>
int launch_main_loop(Kernel kernel, size_t smem, bool ring, const void *a, uint64_t a_rows, unsigned a_cols,
                     const void *b, uint64_t b_rows, unsigned b_cols, unsigned rows, unsigned cols, unsigned batch,
                     Launch launch) {
  constexpr int BK = SemiringTile<T>::BK;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
  if (e != cudaSuccess || a == nullptr) return static_cast<int>(e);
  CUtensorMap tmap_a, tmap_b;
  if ((ring && encode_plain_2d(&tmap_a, a, sizeof(T), a_rows, a_cols, SemiringRing::BM, BK) != 0) ||
      encode_plain_2d(&tmap_b, b, sizeof(T), b_rows, b_cols, BK, BN) != 0) {
    return static_cast<int>(cudaErrorInvalidValue);
  }
  launch(dim3((cols + BN - 1) / BN, (rows + SemiringRing::BM - 1) / SemiringRing::BM, batch), tmap_a, tmap_b);
  return static_cast<int>(cudaGetLastError());
}

// The kernels shaped like the product (plain, accumulate, witness): the ring kernel Kernels::ring_kernel() where it
// serves, else the tile kernel Kernels::tile_kernel() of TN columns per thread, with `extra` (the witness matrix)
// passed after C.  Only the kernels a translation unit launches are instantiated there.
template <typename T, int TN, class Kernels, class... Extra>
int launch_semiring_kernels(const GemmArgs &g, Extra... extra) {
  const GemmBatch &batch = g.batch;
  const unsigned n = g.n, k = g.k, m = g.m, a_step = batch.shared_a ? 0u : 1u, b_step = batch.shared_b ? 0u : 1u;
  const void *a = g.dry_run ? nullptr : g.a;  // null A: load the kernel, launch nothing
  const bool ta = (g.flags & MM_FLAG_TRANSPOSED_A) != 0;
  const uint64_t a_rows = uint64_t(batch.a_copies()) * n, b_rows = uint64_t(batch.b_copies()) * k;
  T *c = static_cast<T *>(g.c);
  if constexpr (sizeof(T) == 4) {
    if (semiring_takes_ring<T>(a, ta, g.tuning ? g.tuning->semiring_ring() : true)) {
      using Cfg = SemiringRing;
      constexpr auto kernel = Kernels::ring_kernel();
      return launch_main_loop<T, Cfg::BN>(
          kernel, Cfg::SMEM_BYTES, true, a, a_rows, k, g.b, b_rows, m, n, m, batch.count,
          [&](dim3 grid, const CUtensorMap &tmap_a, const CUtensorMap &tmap_b) {
            kernel<<<grid, Cfg::THREADS, Cfg::SMEM_BYTES, g.stream>>>(tmap_a, tmap_b, c, extra..., n, k, m, a_step,
                                                                       b_step);
          });
    }
  }
  using Cfg = SemiringTile<T, TN>;
  constexpr auto kernel = Kernels::tile_kernel();
  return launch_main_loop<T, Cfg::BN>(
      kernel, Cfg::SMEM_BYTES, false, a, a_rows, k, g.b, b_rows, m, n, m, batch.count,
      [&](dim3 grid, const CUtensorMap &, const CUtensorMap &tmap_b) {
        kernel<<<grid, Cfg::THREADS, Cfg::SMEM_BYTES, g.stream>>>(static_cast<const T *>(a), tmap_b, c, extra..., n, k,
                                                                   m, ta, a_step, b_step);
      });
}

// The four families of main-loop kernels, each a type with `static int launch(const GemmArgs &, unsigned *w)` per
// (T, Map, Reduce): the product, the accumulate call, the witness call (w: the witness matrix) and the closure.
template <typename T, class Map, class Reduce, bool ACC>
struct SemiringProducts {
  static constexpr auto ring_kernel() {
    if constexpr (ACC) return semiring_accumulate_ring_kernel<T, Map, Reduce>;
    else return semiring_ring_kernel<T, Map, Reduce>;
  }
  static constexpr auto tile_kernel() {
    if constexpr (ACC) return semiring_accumulate_tile_kernel<T, Map, Reduce>;
    else return semiring_tile_kernel<T, Map, Reduce>;
  }
  static int launch(const GemmArgs &g, unsigned *) { return launch_semiring_kernels<T, 8, SemiringProducts>(g); }
};
template <typename T, class Map, class Reduce>
using SemiringProduct = SemiringProducts<T, Map, Reduce, false>;
template <typename T, class Map, class Reduce>
using SemiringAccumulate = SemiringProducts<T, Map, Reduce, true>;
template <typename T, class Map, class Reduce>
struct SemiringWitness;  // semiring_witness_kernel.cuh
template <typename T, class Map, class Reduce>
struct SemiringClosure;  // semiring_closure_kernel.cuh

// One translation unit per (family, data type, map operator) instantiates the family's reduces
// (semiring_*inst.cu compiled with -DMM_INST_T=<type> -DMM_INST_MAP=<MM_OP_*>), so that the small units build in
// parallel and each object holds one family's kernels only.  Returns -1 for a reduce the unit does not hold.
template <template <typename, class, class> class Family, typename T, int MAP_OP>
int launch_semiring_for(int reduce_op, const GemmArgs &g, unsigned *w);

template <template <typename, class, class> class Family, typename T, int MAP_OP, int... REDUCES>
int launch_semiring_reduce(int reduce_op, const GemmArgs &g, unsigned *w) {
  using Map = typename OpSelect<T, MAP_OP>::type;
  int rc = -1;
  (void)((reduce_op == REDUCES &&
          (rc = Family<T, Map, typename OpSelect<T, REDUCES>::type>::launch(g, w), true)) || ...);
  return rc;
}

// The reduces, then for float the FMNMX pair MinFast / MaxFast.
#define MM_INSTANTIATE_SEMIRING(FAMILY, TYPE, MAPOP, ...)                                                           \
  template <>                                                                                                       \
  int launch_semiring_for<FAMILY, TYPE, MAPOP>(int reduce_op, const GemmArgs &g, unsigned *w) {                     \
    if constexpr (std::is_same<TYPE, float>::value) {                                                               \
      return launch_semiring_reduce<FAMILY, TYPE, MAPOP, __VA_ARGS__, MM_OP_MIN_FAST, MM_OP_MAX_FAST>(reduce_op, g, \
                                                                                                      w);           \
    } else {                                                                                                        \
      return launch_semiring_reduce<FAMILY, TYPE, MAPOP, __VA_ARGS__>(reduce_op, g, w);                             \
    }                                                                                                               \
  }

}  // namespace mm
