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
// Phase 3 is the product kernels' main loop (semiring_ring_kernel / semiring_tile_kernel, same per-element order of
// operations) with three differences: the accumulators start from the C tile instead of the reduce's identity, the
// operands are the panels of D read in place with row pitch N (TMA views of the whole batch, or pointers), and the
// k loop covers exactly K_r's width: a multiple of the memory width, so a partial last panel never feeds the
// zero-filled part of a TMA box into a term.  The CTA tile is 128 x 128 = b x b, so the tiles of block row and block
// column r are whole CTAs; they return at once (they would race with the panels they read).  The other tiles read
// only the panels and their own elements, and write only their own.
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

// Phase 3, 4-byte types: the ring kernel's TMA ring over the column panel (A: rows of the tile, columns K_r) and the
// row panel (B: rows K_r, columns of the tile), both views of the whole batch (batch * N rows of N elements).
template <typename T, class Map, class Reduce>
__global__ void __launch_bounds__(256, 2)
semiring_closure_ring_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                             T *__restrict__ D, unsigned n, unsigned r) {
  static_assert(sizeof(T) == 4, "ring variant: 4-byte element types");
  using Cfg = SemiringRing;
  using Term = ClosureTerm<T, Map>;
  constexpr int BM = Cfg::BM, BN = Cfg::BN, BK = Cfg::BK, STAGES = Cfg::STAGES;
  if (blockIdx.x == r || blockIdx.y == r) return;  // block row / column r: the panels themselves
  T *C = D + size_t(blockIdx.z) * n * n;
  const unsigned k0 = r * kClosureBlock, p_row0 = blockIdx.z * n;

  extern __shared__ unsigned char smem_raw[];
  const uint32_t smem0 = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t full0 = smem0 + STAGES * Cfg::STAGE_BYTES, empty0 = full0 + 8 * STAGES;

  const int tid = threadIdx.x, lane = tid % 32;
  const int tx = tid % 16;  // column quad index
  const int ty = tid / 16;  // row quad index
  const unsigned row0 = blockIdx.y * BM, col0 = blockIdx.x * BN;
  const unsigned k_tiles = min(kClosureBlock, n - k0) / BK;  // K_r's width is a multiple of BK: no zero-filled k

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
    ptx::tma_load_2d(as, &tmap_a, bar, int32_t(k0 + kt * BK), int32_t(p_row0 + row0), ptx::L2_EVICT_NORMAL);
    ptx::tma_load_2d(bs, &tmap_b, bar, int32_t(col0), int32_t(p_row0 + k0 + kt * BK), ptx::L2_EVICT_NORMAL);
  };
  if (tid == 0) {
    for (unsigned kt = 0; kt < unsigned(Cfg::AHEAD) && kt < k_tiles; ++kt) load_tile(kt);
  }

  // The seed: this thread's elements of the C tile, in the store's layout (rows past N are never stored).  Element
  // (i, h) of the thread sits at c_thr(n) + c_off(i, h, n).  The epilogue recomputes the addresses and masks from an
  // opaque copy of n, so that they are not kept alive (or spilled) across the main loop.
  auto c_thr = [&](unsigned nn) { return C + size_t(row0 + ty * 4) * nn + col0 + tx * 4; };
  auto c_off = [&](int i, int h, unsigned nn) { return unsigned((i / 4) * 64 + (i % 4)) * nn + h * 64; };
  auto c_in = [&](int i, int h, unsigned nn) {
    return row0 + ty * 4 + (i / 4) * 64 + (i % 4) < nn && col0 + tx * 4 + h * 64 < nn;
  };
  T acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      Quad<T> old;
      if (c_in(i, h, n)) {
        old = *reinterpret_cast<const Quad<T> *>(c_thr(n) + c_off(i, h, n));
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q) old.v[q] = Reduce::identity();
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[i][h * 4 + q] = old.v[q];
    }
  }

  const int r_lo = ty * 4, r_hi = 64 + ty * 4;

  for (unsigned kt = 0; kt < k_tiles; ++kt) {
    const int stage = kt % STAGES;
    if (tid == 0 && kt + Cfg::AHEAD < k_tiles) load_tile(kt + Cfg::AHEAD);
    ptx::mbar_wait(full0 + 8 * stage, (kt / STAGES) & 1);
    const unsigned char *as = smem_raw + (smem0 - ptx::smem_u32(smem_raw)) + stage * Cfg::STAGE_BYTES;
    const T *bs = reinterpret_cast<const T *>(as + Cfg::A_BYTES);

#pragma unroll
    for (int c = 0; c < BK / 4; ++c) {
      T a4[8][4];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int rr = (i < 4 ? r_lo : r_hi) + (i % 4);
        const Quad<T> q = *reinterpret_cast<const Quad<T> *>(as + rr * 64 + c * 16);
#pragma unroll
        for (int v = 0; v < 4; ++v) a4[i][v] = Term::prep(q.v[v]);
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
            bf[u][q] = Term::prep(b0.v[q]);
            bf[u][4 + q] = Term::prep(b1.v[q]);
          }
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            acc[i][j] = Reduce::Apply(Reduce::Apply(acc[i][j], Term::apply(a4[i][kp], bf[0][j])),
                                      Term::apply(a4[i][kp + 1], bf[1][j]));
          }
        }
      }
    }
    __syncwarp();
    if (lane == 0) ptx::mbar_arrive(empty0 + 8 * stage);
  }

  unsigned n_epi;
  asm volatile("mov.u32 %0, %1;" : "=r"(n_epi) : "r"(n));
#pragma unroll
  for (int i = 0; i < 8; ++i) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (c_in(i, h, n_epi)) {
        Quad<T> out;
#pragma unroll
        for (int q = 0; q < 4; ++q) out.v[q] = acc[i][h * 4 + q];
        *reinterpret_cast<Quad<T> *>(c_thr(n_epi) + c_off(i, h, n_epi)) = out;
      }
    }
  }
}

// Phase 3, the other types: the tile kernel's scheme.  The column panel is read through registers (rows clamped to
// N - 1, never stored), transposed into shared memory; the row panel arrives by TMA from the view of the whole batch.
template <typename T, class Map, class Reduce>
__global__ void __launch_bounds__(256, 1)
semiring_closure_tile_kernel(const __grid_constant__ CUtensorMap tmap_b, T *__restrict__ D, unsigned n, unsigned r) {
  using Cfg = SemiringTile<T>;
  using Term = ClosureTerm<T, Map>;
  constexpr int BM = Cfg::BM, BN = Cfg::BN, BK = Cfg::BK, VEC = Cfg::VEC;
  constexpr int LDA = Cfg::LDA, LDB = Cfg::LDB;
  if (blockIdx.x == r || blockIdx.y == r) return;
  T *C = D + size_t(blockIdx.z) * n * n;
  const unsigned k0 = r * kClosureBlock, b_k0 = blockIdx.z * n + k0;
  const T *A = C + k0;  // the column panel: row i at A + i * n

  extern __shared__ __align__(128) unsigned char smem_raw[];
  T *As = reinterpret_cast<T *>(smem_raw);
  T *Bs = reinterpret_cast<T *>(smem_raw + Cfg::A_BYTES);
  const uint32_t bar0 = ptx::smem_u32(smem_raw + Cfg::A_BYTES + 2 * Cfg::B_TILE_BYTES);

  const int tid = threadIdx.x;
  const int tx = tid % 16;
  const int ty = tid / 16;
  const size_t row0 = size_t(blockIdx.y) * BM;
  const size_t col0 = size_t(blockIdx.x) * BN;

  T acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const size_t row = row0 + (i / 4) * 64 + ty * 4 + (i % 4);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const size_t col = col0 + h * 64 + tx * 4;
      Quad<T> old;
      if (row < n && col + 4 <= n) {
        old = *reinterpret_cast<const Quad<T> *>(C + row * n + col);
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q) old.v[q] = Reduce::identity();
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[i][h * 4 + q] = old.v[q];
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
  auto load_b_tma = [&](int buf, unsigned kk0) {
    if (tid == 0) {
      ptx::mbar_arrive_expect_tx(bar0 + 8 * buf, uint32_t(Cfg::B_TILE_BYTES));
      ptx::tma_load_2d(ptx::smem_u32(Bs + buf * BK * LDB), &tmap_b, bar0 + 8 * buf, int32_t(col0), int32_t(b_k0 + kk0),
                       ptx::L2_EVICT_NORMAL);
    }
  };
  auto load_global = [&](unsigned kk0) {
#pragma unroll
    for (int i = 0; i < Cfg::CHUNKS_PER_THREAD; ++i) {
      const int c = tid + i * Cfg::THREADS;
      const int rr = c / Cfg::A_CHUNKS_PER_ROW;
      const int part = c % Cfg::A_CHUNKS_PER_ROW;
      size_t row = row0 + rr;
      if (row >= n) row = n - 1;
      a_stage[i] = *reinterpret_cast<const Chunk16<T> *>(A + row * n + kk0 + part * VEC);
    }
  };
  auto store_shared = [&](int buf) {
    T *as = As + buf * BK * LDA;
#pragma unroll
    for (int i = 0; i < Cfg::CHUNKS_PER_THREAD; ++i) {
      const int c = tid + i * Cfg::THREADS;
      const int rr = c / Cfg::A_CHUNKS_PER_ROW;
      const int part = c % Cfg::A_CHUNKS_PER_ROW;
#pragma unroll
      for (int v = 0; v < VEC; ++v) as[(part * VEC + v) * LDA + rr] = a_stage[i].v[v];
    }
  };

  const unsigned k_tiles = min(kClosureBlock, n - k0) / BK;  // a multiple of the memory width BK
  load_b_tma(0, 0);
  load_global(0);
  store_shared(0);
  __syncthreads();
  ptx::mbar_wait(bar0, 0);

  for (unsigned kt = 0; kt < k_tiles; ++kt) {
    const int buf = kt & 1;
    constexpr bool kRolled = ClosureRolledK<T, Map>::value;
    if (kt + 1 < k_tiles) {
      load_b_tma(buf ^ 1, (kt + 1) * BK);
      if (!kRolled) load_global((kt + 1) * BK);
    }
    const T *as = As + buf * BK * LDA;
    const T *bs = Bs + buf * BK * LDB;
    constexpr int KK_UNROLL = ClosureRolledK<T, Map>::value ? 1 : BK / 2;
#pragma unroll KK_UNROLL
    for (int kk = 0; kk < BK; kk += 2) {
      T af[2][8], bf[2][8];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const Quad<T> a0 = *reinterpret_cast<const Quad<T> *>(as + (kk + u) * LDA + ty * 4);
        const Quad<T> a1 = *reinterpret_cast<const Quad<T> *>(as + (kk + u) * LDA + 64 + ty * 4);
        const Quad<T> b0 = *reinterpret_cast<const Quad<T> *>(bs + (kk + u) * LDB + tx * 4);
        const Quad<T> b1 = *reinterpret_cast<const Quad<T> *>(bs + (kk + u) * LDB + 64 + tx * 4);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          af[u][q] = Term::prep(a0.v[q]);
          af[u][4 + q] = Term::prep(a1.v[q]);
          bf[u][q] = Term::prep(b0.v[q]);
          bf[u][4 + q] = Term::prep(b1.v[q]);
        }
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          acc[i][j] = Reduce::Apply(Reduce::Apply(acc[i][j], Term::apply(af[0][i], bf[0][j])),
                                    Term::apply(af[1][i], bf[1][j]));
        }
      }
    }
    if (kt + 1 < k_tiles) {
      if (kRolled) load_global((kt + 1) * BK);
      store_shared(buf ^ 1);
    }
    __syncthreads();
    if (kt + 1 < k_tiles) ptx::mbar_wait(bar0 + 8 * (buf ^ 1), ((kt + 1) >> 1) & 1u);
  }

#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const size_t row = row0 + (i / 4) * 64 + ty * 4 + (i % 4);
    if (row >= n) continue;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const size_t col = col0 + h * 64 + tx * 4;
      if (col + 4 <= n) {
        Quad<T> out;
#pragma unroll
        for (int q = 0; q < 4; ++q) out.v[q] = acc[i][h * 4 + q];
        *reinterpret_cast<Quad<T> *>(C + row * n + col) = out;
      }
    }
  }
}

// Host side: every round of the closure of `batch` packed N x N problems at d, on one stream.  Returns a cudaError_t
// value as int.
template <typename T, class Map, class Reduce>
int launch_semiring_closure_typed(void *d, unsigned n, unsigned batch, cudaStream_t stream) {
  T *D = static_cast<T *>(d);
  const unsigned blocks = (n + kClosureBlock - 1) / kClosureBlock;
  const size_t panel_smem = ClosureStep::diag_bytes<T>();
  cudaError_t e = cudaFuncSetAttribute(semiring_closure_panel_kernel<T, Map, Reduce>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, int(panel_smem));
  if (e != cudaSuccess) return static_cast<int>(e);
  // both panels are read in place through a view of the whole batch: batch * N rows of N elements
  const uint64_t rows = uint64_t(batch) * n;
  CUtensorMap tmap_a, tmap_b;
  size_t phase3_smem;
  if constexpr (sizeof(T) == 4) {
    using Cfg = SemiringRing;
    phase3_smem = Cfg::SMEM_BYTES;
    e = cudaFuncSetAttribute(semiring_closure_ring_kernel<T, Map, Reduce>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             int(phase3_smem));
    if (e != cudaSuccess) return static_cast<int>(e);
    if (encode_plain_2d(&tmap_a, d, sizeof(T), rows, n, Cfg::BM, Cfg::BK) != 0 ||
        encode_plain_2d(&tmap_b, d, sizeof(T), rows, n, Cfg::BK, Cfg::BN) != 0) {
      return static_cast<int>(cudaErrorInvalidValue);
    }
  } else {
    using Cfg = SemiringTile<T>;
    phase3_smem = Cfg::SMEM_BYTES;
    if (encode_plain_2d(&tmap_b, d, sizeof(T), rows, n, Cfg::BK, Cfg::BN) != 0) {
      return static_cast<int>(cudaErrorInvalidValue);
    }
  }
  const dim3 block(ClosureStep::THREADS);
  for (unsigned r = 0; r < blocks; ++r) {
    semiring_closure_pivot_kernel<T, Map, Reduce><<<dim3(1, 1, batch), block, 0, stream>>>(D, n, r);
    if (blocks == 1) break;  // no panels, no remainder
    semiring_closure_panel_kernel<T, Map, Reduce><<<dim3(blocks, 2, batch), block, panel_smem, stream>>>(D, n, r);
    const dim3 grid(blocks, blocks, batch);
    if constexpr (sizeof(T) == 4) {
      semiring_closure_ring_kernel<T, Map, Reduce><<<grid, block, phase3_smem, stream>>>(tmap_a, tmap_b, D, n, r);
    } else {
      semiring_closure_tile_kernel<T, Map, Reduce><<<grid, block, phase3_smem, stream>>>(tmap_b, D, n, r);
    }
  }
  return static_cast<int>(cudaGetLastError());
}

// One translation unit per (data type, map operator) instantiates the Min / Max reduces, plus the FMNMX pair for
// float (semiring_closure_inst.cu compiled with -DMM_INST_T=<type> -DMM_INST_MAP=<MM_OP_*>).
template <typename T, int MAP_OP>
int launch_semiring_closure_for(int reduce_op, void *d, unsigned n, unsigned batch, cudaStream_t stream);

#define MM_CLOSURE_CASE(REDOP)                                                                      \
  if (reduce_op == REDOP)                                                                           \
    return launch_semiring_closure_typed<T, typename OpSelect<T, MAP_OP>::type,                     \
                                         typename OpSelect<T, REDOP>::type>(d, n, batch, stream);

#define MM_INSTANTIATE_SEMIRING_CLOSURE(TYPE, MAPOP)                                                \
  template <>                                                                                       \
  int launch_semiring_closure_for<TYPE, MAPOP>(int reduce_op, void *d, unsigned n, unsigned batch,  \
                                               cudaStream_t stream) {                               \
    using T = TYPE;                                                                                 \
    constexpr int MAP_OP = MAPOP;                                                                   \
    MM_CLOSURE_CASE(MM_OP_MIN)                                                                      \
    MM_CLOSURE_CASE(MM_OP_MAX)                                                                      \
    if constexpr (std::is_same<T, float>::value) {                                                  \
      MM_CLOSURE_CASE(MM_OP_MIN_FAST)                                                               \
      MM_CLOSURE_CASE(MM_OP_MAX_FAST)                                                               \
    }                                                                                               \
    return -1;                                                                                      \
  }

}  // namespace mm
