// Witness variants of the CUDA-core semiring kernels (mm_kernel_enqueue_witness): C exactly as
// semiring_tile_kernel / semiring_ring_kernel compute it, and beside every accumulator a uint32 register holding
// the last k at which the Min / Max reduction selected its new term (MM_WITNESS_NONE if it never did).
//
// Both kernels run the product kernels' main loops (semiring_tile_body, semiring_ring_body) with WitnessVariant,
// which supplies the seed (the reduce's identity, MM_WITNESS_NONE witnesses), the element step and the epilogue.  The
// step computes t = Map(a, b) once, decides Selects<Reduce>::apply(acc, t), applies Reduce::Apply(acc, t) (FMNMX stays
// FMNMX on the float default, so C keeps its bits) and moves k into the witness when the term was selected.  The two
// k of a pair are processed in order, k then k + 1, as Naive<> does.
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

// One element-step: t = Map(a, b); the witness takes k when Reduce selects t.
template <class Map, class Reduce, typename T>
__device__ __forceinline__ void witness_step(T &acc, unsigned &w, T a, T b, unsigned k) {
  const T t = Map::Apply(a, b);
  const bool s = Selects<Reduce>::apply(acc, t);
  acc = Reduce::Apply(acc, t);
  w = s ? k : w;
}

// TN columns per thread: 8 in the ring kernel, 4 (one quad, a 128 x 64 CTA tile, k loop rolled) in the tile kernel.
// W: problem 0's witness matrix, laid out as C.
template <typename T, class Map, class Reduce, int TN_>
struct WitnessVariant : SemiringVariant<T, Map, Reduce> {
  static constexpr int TN = TN_;
  static constexpr bool kRolledK = TN_ == 4, kFinish = true;
  using State = unsigned;  // the witness
  unsigned *W;
  __device__ __forceinline__ WitnessVariant(T *c, unsigned *w, unsigned n, unsigned m)
      : SemiringVariant<T, Map, Reduce>{c, n, m}, W(w) {}

  template <typename I>
  __device__ __forceinline__ void seed(T (&acc)[8][TN], unsigned (&wit)[8][TN], T *, I, I, int, int) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int j = 0; j < TN; ++j) {
        acc[i][j] = Reduce::identity();
        wit[i][j] = MM_WITNESS_NONE;
      }
    }
  }

  __device__ __forceinline__ T step(const T &acc, unsigned &w, const T &a0, const T &b0, const T &a1, const T &b1,
                                    unsigned k) {
    T r = acc;
    witness_step<Map, Reduce>(r, w, a0, b0, k);
    witness_step<Map, Reduce>(r, w, a1, b1, k + 1);
    return r;
  }

  // C and W under C's mask (row < N, col + 4 <= M), in 16-byte stores.
  template <typename I>
  __device__ __forceinline__ void finish(const T (&acc)[8][TN], const unsigned (&wit)[8][TN], I row0, I col0,
                                         int tx, int ty) {
    const unsigned size_n = this->size_n, size_m = this->size_m;
    T *C = this->C + size_t(blockIdx.z) * size_n * size_m;
    unsigned *w = W + size_t(blockIdx.z) * size_n * size_m;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const size_t row = size_t(row0) + ((i / 4) * 64 + ty * 4 + (i % 4));
      if (row >= size_n) continue;
#pragma unroll
      for (int h = 0; h < TN / 4; ++h) {
        const size_t col = size_t(col0) + (h * 64 + tx * 4);
        if (col + 4 <= size_m) {
          Quad<T> out;
#pragma unroll
          for (int q = 0; q < 4; ++q) out.v[q] = acc[i][h * 4 + q];
          *reinterpret_cast<Quad<T> *>(C + row * size_m + col) = out;
          *reinterpret_cast<uint4 *>(w + row * size_m + col) =
              make_uint4(wit[i][h * 4], wit[i][h * 4 + 1], wit[i][h * 4 + 2], wit[i][h * 4 + 3]);
        }
      }
    }
  }
};

// Register-staged witness kernel: every type, A row-major or stored K x N.
template <typename T, class Map, class Reduce>
__global__ void __launch_bounds__(256, 1)
semiring_witness_tile_kernel(const T *__restrict__ A, const __grid_constant__ CUtensorMap tmap_b, T *__restrict__ C,
                             unsigned *__restrict__ W, unsigned size_n, unsigned size_k, unsigned size_m,
                             bool TRANSPOSED_A, unsigned a_step, unsigned b_step) {
  semiring_tile_body(WitnessVariant<T, Map, Reduce, 4>(C, W, size_n, size_m), A, a_step, size_k, TRANSPOSED_A, tmap_b,
                     b_step, size_k, 0u);
}

// TMA-ring witness kernel: 4-byte types, A row-major.
template <typename T, class Map, class Reduce>
__global__ void __launch_bounds__(256, 1)
semiring_witness_ring_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                             T *__restrict__ C, unsigned *__restrict__ W, unsigned size_n, unsigned size_k,
                             unsigned size_m, unsigned a_step, unsigned b_step) {
  semiring_ring_body(WitnessVariant<T, Map, Reduce, 8>(C, W, size_n, size_m), tmap_a, a_step, 0u, tmap_b, b_step,
                     size_k, 0u);
}

// Host side: the product's kernel choice and launch, with W after C.
template <typename T, class Map, class Reduce>
struct SemiringWitness {
  static constexpr auto ring_kernel() { return semiring_witness_ring_kernel<T, Map, Reduce>; }
  static constexpr auto tile_kernel() { return semiring_witness_tile_kernel<T, Map, Reduce>; }
  static int launch(const GemmArgs &g, unsigned *w) { return launch_semiring_kernels<T, 4, SemiringWitness>(g, w); }
};

}  // namespace mm
