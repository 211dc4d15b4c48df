// Closure of square matrices over a Min / Max semiring, in place, by blocked Floyd–Warshall
// (mm_kernel_enqueue_closure).  D is `batch` packed N x N row-major problems; blocks of
// b = kClosureBlock indices K_r = [r*b, min((r+1)*b, N)); round r = 0, 1, ... runs three kernels on one stream:
//
//   1. semiring_closure_pivot_kernel  (one CTA per problem): for k in K_r ascending, step k over the diagonal
//      block K_r x K_r;
//   2. semiring_closure_panel_kernel  (one CTA per (block J != r, panel, problem)): for k in K_r ascending, step k
//      over the row panel K_r x J and the column panel J x K_r, reading the finished diagonal block;
//   3. semiring_closure_ring_kernel (4-byte types) / semiring_closure_tile_kernel (the others): every tile outside
//      block row and block column r gets D[i][j] <- R(...R(R(D[i][j], t_k0), t_k0+1)..., t_klast), t_k =
//      Map(D[i][k], D[k][j]), the k running over K_r in order: a rank-b update seeded with D itself.
//
// A step k updates its elements simultaneously: D'[i][j] = R(D[i][j], Map(D[i][k], D[k][j])) with every read seeing
// the values from before the step.  Phases 1 and 2 keep their block in registers (16 x 16 threads, 8 x 8 elements
// each); before each step the owners of row k and column k publish them to shared memory, one barrier, and every
// thread updates its 64 elements from the published copies.  The copies alternate between two buffers by the parity
// of k, so a step needs one barrier: a buffer is rewritten two steps later, after every thread has passed the barrier
// that follows its last read.
//
// Phase 3 runs the product kernels' main loops (semiring_ring_body / semiring_tile_body, so the per-element order of
// operations is theirs) with a closure variant: the accumulators start from the C tile instead of the reduce's
// identity, the operands are the panels of D read in place with row pitch N (TMA views of the whole batch, or
// pointers), and the k loop covers exactly K_r's width: a multiple of the memory width, so a partial last panel never
// feeds the zero-filled part of a TMA box into a term.  The CTA tile is 128 x 128 = b x b, so the tiles of block row
// and block column r are whole CTAs; they return at once (they would race with the panels they read).  The other tiles
// read only the panels and their own elements, and write only their own.
#pragma once

#include "semiring_kernel.cuh"

namespace mm {

constexpr unsigned kClosureBlock = 128;  // b: every type (the double diagonal block takes 128 KiB of shared memory)

struct ClosureStep {
  static constexpr int B = int(kClosureBlock), THREADS = 256, R = 8;  // 16 x 16 threads of R x R elements
  template <typename T>
  static constexpr size_t diag_bytes() {  // phase 2: the finished diagonal block
    return size_t(B) * B * sizeof(T);
  }
};
static_assert(ClosureStep::B == SemiringRing::BM && ClosureStep::B == SemiringRing::BN, "b is the CTA tile");
static_assert(ClosureStep::B == SemiringTile<float>::BM && ClosureStep::B == SemiringTile<float>::BN, "b is the CTA tile");

// uint8_t with an And Map keeps phase 3's k loop rolled (one pair of k per iteration) and loads the next tile of the
// column panel after the compute, not before: unrolled, with the staged tile live, ptxas hoists the data-independent
// And terms far ahead and spills kilobytes, as in the plain and witness kernels.
template <typename T, class Map>
struct ClosureRolledK {
  static constexpr bool value = std::is_same<Map, And<T>>::value && sizeof(T) == 1;
};

// The term Map(a, b) of every phase as prep(a) (x) prep(b).  For an And Map, prep(x) = And(x, 1) is 0 or 1 and the
// term is the product of the two in T: exactly And(a, b), bit for bit in every type (+0 or 1), without the compare
// and select per term that made ptxas hoist the terms and spill.  Every other Map is applied as it is.
template <typename T, class Map>
struct ClosureTerm {
  static __device__ __forceinline__ T prep(T x) { return x; }
  static __device__ __forceinline__ T apply(T a, T b) { return Map::Apply(a, b); }
};
template <typename T>
struct ClosureTerm<T, And<T>> {
  static __device__ __forceinline__ T prep(T x) { return And<T>::Apply(x, Prim<T>::one()); }
  static __device__ __forceinline__ T apply(T a, T b) { return Prim<T>::mul(a, b); }
};

// The steps k = 0 .. wk-1 (pivot-local) over one register-held block.  MODE 0: the diagonal block (both operands
// from the block itself); 1: a row panel K_r x J (D[i][k] from the diagonal block in shared memory, D[k][j] from the
// panel); 2: a column panel J x K_r (D[i][k] from the panel, D[k][j] from the diagonal block).
template <typename T, class Map, class Reduce, int MODE>
__device__ __forceinline__ void closure_steps(T (&v)[8][8], const T *diag_s, unsigned wk) {
  constexpr int B = ClosureStep::B, R = ClosureStep::R;
  using Term = ClosureTerm<T, Map>;
  __shared__ __align__(16) T col_s[2][B];  // D[i][k] of this step, by block row i
  __shared__ __align__(16) T row_s[2][B];  // D[k][j] of this step, by block column j
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  // One step per iteration, not unrolled: the owners pick their row / column kr of v by compare and select, so v
  // stays in registers, and ptxas has no later step's terms to hoist (with the steps unrolled, an And Map spilled).
#pragma unroll 1
  for (unsigned k = 0; k < wk; ++k) {
    const int kt = k / R, kr = k % R, buf = k & 1;
    if (MODE != 1 && tx == kt) {
#pragma unroll
      for (int i = 0; i < R; ++i) {
        T x = v[i][0];
#pragma unroll
        for (int c = 1; c < R; ++c) x = (c == kr) ? v[i][c] : x;
        col_s[buf][ty * R + i] = x;
      }
    }
    if (MODE != 2 && ty == kt) {
#pragma unroll
      for (int j = 0; j < R; ++j) {
        T x = v[0][j];
#pragma unroll
        for (int c = 1; c < R; ++c) x = (c == kr) ? v[c][j] : x;
        row_s[buf][tx * R + j] = x;
      }
    }
    __syncthreads();
    T a[R], b[R];
#pragma unroll
    for (int i = 0; i < R; ++i) a[i] = Term::prep(MODE == 1 ? diag_s[(ty * R + i) * B + k] : col_s[buf][ty * R + i]);
#pragma unroll
    for (int j = 0; j < R; ++j) b[j] = Term::prep(MODE == 2 ? diag_s[k * B + tx * R + j] : row_s[buf][tx * R + j]);
#pragma unroll
    for (int i = 0; i < R; ++i) {
#pragma unroll
      for (int j = 0; j < R; ++j) v[i][j] = Reduce::Apply(v[i][j], Term::apply(a[i], b[j]));
    }
  }
}

// The block of h x w elements at p (row pitch n) to and from the registers of closure_steps; elements outside it
// (a partial last block) take the reduce's identity, are updated like the others and never stored.
template <typename T, class Reduce>
__device__ __forceinline__ void closure_load(T (&v)[8][8], const T *p, unsigned n, unsigned h, unsigned w) {
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const unsigned r = ty * 8 + i, c = tx * 8 + j;
      v[i][j] = (r < h && c < w) ? p[size_t(r) * n + c] : Reduce::identity();
    }
  }
}
template <typename T>
__device__ __forceinline__ void closure_store(const T (&v)[8][8], T *p, unsigned n, unsigned h, unsigned w) {
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const unsigned r = ty * 8 + i, c = tx * 8 + j;
      if (r < h && c < w) p[size_t(r) * n + c] = v[i][j];
    }
  }
}

// Phase 1: grid (1, 1, batch).
template <typename T, class Map, class Reduce>
__global__ void __launch_bounds__(256, 1) semiring_closure_pivot_kernel(T *__restrict__ D, unsigned n, unsigned r) {
  const unsigned k0 = r * kClosureBlock, wk = min(kClosureBlock, n - k0);
  T *p = D + size_t(blockIdx.z) * n * n + size_t(k0) * n + k0;
  T v[8][8];
  closure_load<T, Reduce>(v, p, n, wk, wk);
  closure_steps<T, Map, Reduce, 0>(v, nullptr, wk);
  closure_store(v, p, n, wk, wk);
}

// Phase 2: grid (blocks, 2, batch); blockIdx.x = J (J == r returns), blockIdx.y = 0 row panel, 1 column panel.
template <typename T, class Map, class Reduce>
__global__ void __launch_bounds__(256, 1) semiring_closure_panel_kernel(T *__restrict__ D, unsigned n, unsigned r) {
  constexpr int B = ClosureStep::B;
  if (blockIdx.x == r) return;
  const unsigned k0 = r * kClosureBlock, wk = min(kClosureBlock, n - k0);
  const unsigned j0 = blockIdx.x * kClosureBlock, wj = min(kClosureBlock, n - j0);
  T *d = D + size_t(blockIdx.z) * n * n;
  extern __shared__ __align__(16) unsigned char closure_smem[];
  T *diag_s = reinterpret_cast<T *>(closure_smem);  // [B][B]; rows / columns past wk are never read
  for (unsigned e = threadIdx.x; e < unsigned(B) * B; e += ClosureStep::THREADS) {
    const unsigned i = e / B, j = e % B;
    if (i < wk && j < wk) diag_s[e] = d[size_t(k0 + i) * n + k0 + j];
  }
  __syncthreads();
  T v[8][8];
  if (blockIdx.y == 0) {
    T *p = d + size_t(k0) * n + j0;
    closure_load<T, Reduce>(v, p, n, wk, wj);
    closure_steps<T, Map, Reduce, 1>(v, diag_s, wk);
    closure_store(v, p, n, wk, wj);
  } else {
    T *p = d + size_t(j0) * n + k0;
    closure_load<T, Reduce>(v, p, n, wj, wk);
    closure_steps<T, Map, Reduce, 2>(v, diag_s, wk);
    closure_store(v, p, n, wj, wk);
  }
}

// Phase 3's variants: problem 0's C is D, with N x N problems; the term is ClosureTerm's; the loop covers at most b k;
// the accumulators start from this thread's elements of the C tile, the reduce's identity outside it.
//
// The ring variant recomputes the addresses of its epilogue from an opaque copy of n, so that they are not kept alive
// (or spilled) across the main loop: element (i, h) of the thread sits at at(C, ..., i, h, n).
template <typename T, class Map, class Reduce>
struct ClosureRingVariant : SemiringVariant<T, Map, Reduce, false, ClosureTerm<T, Map>> {
  static constexpr bool kFinish = true;
  static constexpr unsigned kMaxK = kClosureBlock;
  template <typename P>
  static __device__ __forceinline__ P *at(P *C, unsigned row0, unsigned col0, int tx, int ty, int i, int h,
                                          unsigned nn) {
    return C + size_t(row0 + ty * 4) * nn + col0 + tx * 4 + (unsigned((i / 4) * 64 + (i % 4)) * nn + h * 64);
  }
  static __device__ __forceinline__ bool in(unsigned row0, unsigned col0, int tx, int ty, int i, int h, unsigned nn) {
    return row0 + ty * 4 + (i / 4) * 64 + (i % 4) < nn && col0 + tx * 4 + h * 64 < nn;
  }

  __device__ __forceinline__ void seed(T (&acc)[8][8], NoState (&)[8][8], const T *C, unsigned row0, unsigned col0,
                                       int tx, int ty) {
    const unsigned n = this->size_n;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        Quad<T> old;
        if (in(row0, col0, tx, ty, i, h, n)) {
          old = *reinterpret_cast<const Quad<T> *>(at(C, row0, col0, tx, ty, i, h, n));
        } else {
#pragma unroll
          for (int q = 0; q < 4; ++q) old.v[q] = Reduce::identity();
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[i][h * 4 + q] = old.v[q];
      }
    }
  }

  __device__ __forceinline__ void finish(const T (&acc)[8][8], NoState (&)[8][8], unsigned row0, unsigned col0,
                                         int tx, int ty) {
    unsigned n_epi;
    asm volatile("mov.u32 %0, %1;" : "=r"(n_epi) : "r"(this->size_n));
    T *C = this->C + size_t(blockIdx.z) * n_epi * n_epi;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (in(row0, col0, tx, ty, i, h, n_epi)) {
          Quad<T> out;
#pragma unroll
          for (int q = 0; q < 4; ++q) out.v[q] = acc[i][h * 4 + q];
          *reinterpret_cast<Quad<T> *>(at(C, row0, col0, tx, ty, i, h, n_epi)) = out;
        }
      }
    }
  }
};

// The tile variant takes the body's C-tile seed and store; uint8_t with an And Map keeps the k loop rolled and loads
// the next tile of the column panel late (ClosureRolledK).
template <typename T, class Map, class Reduce>
struct ClosureTileVariant : SemiringVariant<T, Map, Reduce, false, ClosureTerm<T, Map>> {
  static constexpr bool kRolledK = ClosureRolledK<T, Map>::value, kLateA = kRolledK, kSeedC = true;
  static constexpr unsigned kMaxK = kClosureBlock;
};

// Phase 3, 4-byte types: the ring's main loop over the column panel (A: rows of the tile, columns K_r) and the row
// panel (B: rows K_r, columns of the tile), both read through views of the whole batch (batch * N rows of N elements).
template <typename T, class Map, class Reduce>
__global__ void __launch_bounds__(256, 2)
semiring_closure_ring_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                             T *__restrict__ D, unsigned n, unsigned r) {
  if (blockIdx.x == r || blockIdx.y == r) return;  // block row / column r: the panels themselves
  const unsigned k0 = r * kClosureBlock;  // K_r's width, min(b, n - k0), is a multiple of BK: no zero-filled k
  semiring_ring_body(ClosureRingVariant<T, Map, Reduce>{{D, n, n}}, tmap_a, 1u, k0, tmap_b, 1u, n, k0);
}

// Phase 3, the other types: the tile's main loop.  The column panel (row i of problem 0 at D + k0 + i * n) is read
// through registers, rows clamped to N - 1 (never stored); the row panel arrives by TMA from the view of the batch.
template <typename T, class Map, class Reduce>
__global__ void __launch_bounds__(256, 1)
semiring_closure_tile_kernel(const __grid_constant__ CUtensorMap tmap_b, T *__restrict__ D, unsigned n, unsigned r) {
  if (blockIdx.x == r || blockIdx.y == r) return;
  const unsigned k0 = r * kClosureBlock;
  semiring_tile_body(ClosureTileVariant<T, Map, Reduce>{{D, n, n}}, D + k0, 1u, n, false, tmap_b, 1u, n, k0);
}

// Host side: every round of the closure of g.batch.count packed N x N problems at g.c, on one stream.  Phase 3 of a
// 4-byte type always takes the ring (D is row-major and 16-byte aligned; there is no tile kernel for it).
template <typename T, class Map, class Reduce>
struct SemiringClosure {
  static int launch(const GemmArgs &g, unsigned *) {
    T *D = static_cast<T *>(g.c);
    const unsigned n = g.n, batch = g.batch.count, blocks = (n + kClosureBlock - 1) / kClosureBlock;
    const size_t panel_smem = ClosureStep::diag_bytes<T>();
    cudaError_t e = cudaFuncSetAttribute(semiring_closure_panel_kernel<T, Map, Reduce>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, int(panel_smem));
    if (e != cudaSuccess) return static_cast<int>(e);
    const dim3 block(ClosureStep::THREADS);
    auto rounds = [&](auto phase3) {
      for (unsigned r = 0; r < blocks; ++r) {
        semiring_closure_pivot_kernel<T, Map, Reduce><<<dim3(1, 1, batch), block, 0, g.stream>>>(D, n, r);
        if (blocks == 1) break;  // no panels, no remainder
        semiring_closure_panel_kernel<T, Map, Reduce><<<dim3(blocks, 2, batch), block, panel_smem, g.stream>>>(D, n, r);
        phase3(r);
      }
    };
    // both panels are read in place through a view of the whole batch: batch * N rows of N elements
    const uint64_t rows = uint64_t(batch) * n;
    if constexpr (sizeof(T) == 4) {
      using Cfg = SemiringRing;
      constexpr auto kernel = semiring_closure_ring_kernel<T, Map, Reduce>;
      return launch_main_loop<T, Cfg::BN>(kernel, Cfg::SMEM_BYTES, true, D, rows, n, D, rows, n, n, n, batch,
                                          [&](dim3 grid, const CUtensorMap &tmap_a, const CUtensorMap &tmap_b) {
                                            rounds([&](unsigned r) {
                                              kernel<<<grid, block, Cfg::SMEM_BYTES, g.stream>>>(tmap_a, tmap_b, D, n,
                                                                                                  r);
                                            });
                                          });
    } else {
      using Cfg = SemiringTile<T>;
      constexpr auto kernel = semiring_closure_tile_kernel<T, Map, Reduce>;
      return launch_main_loop<T, Cfg::BN>(kernel, Cfg::SMEM_BYTES, false, D, rows, n, D, rows, n, n, n, batch,
                                          [&](dim3 grid, const CUtensorMap &, const CUtensorMap &tmap_b) {
                                            rounds([&](unsigned r) {
                                              kernel<<<grid, block, Cfg::SMEM_BYTES, g.stream>>>(tmap_b, D, n, r);
                                            });
                                          });
    }
  }
};

}  // namespace mm
