// The DMMA GEMM kernel for double and its launcher, shared by gemm_dmma.cu (the plain kernels) and gemm_dmma_acc.cu
// (the accumulate kernels of mm_kernel_enqueue_accumulate).
//
// Tensor-core path for the dense (Multiply, Add) contraction on double:  C = A * B  in FP64.
// wgmma has no f64 kind, so this is the warp-level DMMA instruction
// mma.sync.aligned.m8n8k4.row.col.f64 (the only FP64 shape sm_90a executes natively; the larger
// PTX shapes are split into it) fed from a TMA shared-memory ring.
// sm_90a counterpart of the reference's PE chain for MM_DATA_TYPE=double
// (kernel/Compute.cpp:53-146; README.md:8 quotes 132 GFLOP/s for it on a VCU1525).
//
// CTA tile BM x 128 (BM = 128, or 64 for short row blocks), BK = 32, 3 stages.  Eight compute warps as
// 2 (rows) x 4 (cols), warp tile (BM / 2) x 32 = MI x 4 m8n8 accumulator tiles (64 doubles per thread
// at BM = 128), plus one producer warp of which a single thread issues the TMA loads.  Stages are
// handed over through mbarriers (full[s]: TMA transaction bytes; empty[s]: one arrival per compute
// warp), so compute warps never meet at a block-wide barrier.
//
// The loads are TMA rather than cp.async (LDGSTS) issued by the compute warps: TMA removes the LSU
// instructions and the address arithmetic from the warps that feed the DMMA pipe.
#pragma once

#include <cuda_runtime.h>

#include <cmath>
#include <cstdlib>
#include <cstdint>

#include "common.cuh"
#include "ptx_sm90.cuh"
#include "tma_host.cuh"

namespace mm {
namespace {

using ptx::fence_mbar_init;
using ptx::mbar_arrive;
using ptx::mbar_init;
using ptx::mbar_wait;
using ptx::smem_u32;

constexpr int BN = 128, BK = 32;
constexpr int STAGES = 3;  // 3 x (32 + 32) KiB at BM = 128

__device__ __forceinline__ void dmma_m8n8k4(double &c0, double &c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

// ---- shared-memory layout -----------------------------------------------------------------------
// TMA writes dense tiles, so bank conflicts are avoided by the 128-byte swizzle (16-byte chunk
// index XOR (tile row % 8)) plus a permutation of which physical rows / columns the eight row- or
// column-slots g of an m8n8k4 fragment stand for (k stays natural: step s, slot q <-> k = 4 s + q):
//   * A row-major: tiles of [BM rows][16 k]; accumulator tile i, slot g <-> row 2 g + (i % 2) + 16 (i / 2):
//     the four rows of a half-warp have row % 8 = {0,2,4,6} (+ i % 2), which XORs the two chunks a
//     row's four k-slots touch onto four disjoint aligned chunk pairs
//   * B (and A when stored K x N): tiles of [32 k][16 columns]; tile j, slot g <-> column
//     (g % 2) + 2 (g / 4) + 8 ((g / 2) % 2) + 4 (j % 2) + 16 (j / 2): a half-warp touches chunks c and
//     c ^ 4, which stay disjoint under the XOR with k % 8 = 4 (s % 2) + q
// Every half-warp LDS.64 then reads sixteen distinct 8-byte words of one 128-byte bank row.
constexpr int TMA_WM = 2, TMA_WN = 4;

// Batch: blockIdx.z = problem.  B (K x M) and A stored K x N can be read past K (BK = 32, K % 8 == 0),
// so their maps are 3-D {columns, K, problems} and zero-fill per problem; row-major A is a 2-D map with
// the problems stacked along the rows (reading past N only feeds rows of C that are never stored).
// a_step / b_step: 1 = packed operands, 0 = every problem reads problem 0's.
// ACC: C = C_old + product, one __dadd_rn per element in the epilogue (gemm_dmma_accumulate_kernel).
template <bool TRANSPOSED_A, int BM, bool ACC>
__device__ __forceinline__ void gemm_dmma_body(const CUtensorMap &map_a, const CUtensorMap &map_b,
                                               double *__restrict__ C, unsigned size_n, unsigned size_k,
                                               unsigned size_m, unsigned a_step, unsigned b_step) {
  constexpr int WM = TMA_WM, WN = TMA_WN, NCW = WM * WN;
  constexpr int MI = BM / (WM * 8), NJ = BN / (WN * 8);
  constexpr int WROWS = BM / WM;  // rows of C per warp
  constexpr uint32_t A_BYTES = BM * BK * 8, B_BYTES = BK * BN * 8, STAGE_BYTES = A_BYTES + B_BYTES;
  extern __shared__ unsigned char smem_raw[];
  const uint32_t smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;  // swizzle atoms are 1024-byte aligned
  const uint32_t full0 = smem0 + STAGES * STAGE_BYTES, empty0 = full0 + 8 * STAGES;

  const int tid = threadIdx.x;
  const int warp = tid / 32, lane = tid % 32;
  const unsigned row0 = blockIdx.y * BM, col0 = blockIdx.x * BN;
  const unsigned k_tiles = (size_k + BK - 1) / BK;

  if (tid == 0) {
    ptx::prefetch_tensormap(&map_a);
    ptx::prefetch_tensormap(&map_b);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, NCW);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == NCW) {
    if (lane != 0) return;
    const int a_prob = int(blockIdx.z * a_step), b_prob = int(blockIdx.z * b_step);
    for (unsigned kt = 0; kt < k_tiles; ++kt) {
      const int stage = kt % STAGES;
      if (kt >= STAGES) mbar_wait(empty0 + 8 * stage, ((kt / STAGES) - 1) & 1);
      const uint32_t as = smem0 + stage * STAGE_BYTES, bs = as + A_BYTES, bar = full0 + 8 * stage;
      const int k0 = int(kt * BK);
      ptx::mbar_arrive_expect_tx(bar, STAGE_BYTES);
      if (!TRANSPOSED_A) {
        const int a_row = a_prob * int(size_n) + int(row0);
#pragma unroll
        for (int kh = 0; kh < BK / 16; ++kh)
          ptx::tma_load_2d(as + kh * BM * 128, &map_a, bar, k0 + kh * 16, a_row, ptx::L2_EVICT_NORMAL);
      } else {
#pragma unroll
        for (int sl = 0; sl < BM / 16; ++sl)
          ptx::tma_load_3d(as + sl * 4096, &map_a, bar, int(row0) + sl * 16, k0, a_prob, ptx::L2_EVICT_NORMAL);
      }
#pragma unroll
      for (int sl = 0; sl < BN / 16; ++sl)
        ptx::tma_load_3d(bs + sl * 4096, &map_b, bar, int(col0) + sl * 16, k0, b_prob, ptx::L2_EVICT_NORMAL);
    }
    return;
  }
  C += size_t(blockIdx.z) * size_n * size_m;

  const int wr = warp / WN, wc = warp % WN;
  const int g = lane / 4, q = lane % 4;
  double acc[MI][NJ][2];
#pragma unroll
  for (int i = 0; i < MI; ++i)
#pragma unroll
    for (int j = 0; j < NJ; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;

  // slot permutation within a 16-wide tile (see above); t16(x) for x = i or j
  const int perm16 = (g % 2) + 2 * (g / 4) + 8 * ((g / 2) % 2);
  // physical row (within the CTA tile) of accumulator tile i, row-slot g
  auto c_row = [&](int i) {
    return TRANSPOSED_A ? wr * WROWS + 16 * (i / 2) + 4 * (i % 2) + perm16
                        : wr * WROWS + 16 * (i / 2) + (i % 2) + 2 * g;
  };
  auto lds = [](uint32_t addr) {
    double v;
    asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(addr));
    return v;
  };

  // Fragment addresses = (stage base + per-thread base + compile-time tile offset) XOR a compile-time
  // chunk constant: everything below bit 7 of the per-thread bases is the thread's own swizzle term,
  // all tile offsets are multiples of 128, so the 16-byte-chunk XOR can be applied to the sum.
  const uint32_t sw_base = q * 128 + (((perm16 / 2) ^ q) * 16) + (perm16 % 2) * 8;  // [32 k][16] tiles
  const uint32_t a_base = TRANSPOSED_A ? (wr * WROWS / 16) * 4096 + sw_base
                                       : (wr * WROWS + 2 * g) * 128 + (((q / 2) ^ ((2 * g) % 8)) * 16) + (q % 2) * 8;
  const uint32_t b_base = wc * (NJ / 2) * 4096 + sw_base;

  for (unsigned kt = 0; kt < k_tiles; ++kt) {
    const int stage = kt % STAGES;
    mbar_wait(full0 + 8 * stage, (kt / STAGES) & 1);
    const uint32_t as = smem0 + stage * STAGE_BYTES + a_base, bs = smem0 + stage * STAGE_BYTES + A_BYTES + b_base;
#pragma unroll
    for (int s = 0; s < BK / 4; ++s) {
      double af[MI], bf[NJ];
#pragma unroll
      for (int i = 0; i < MI; ++i) {
        if (!TRANSPOSED_A) {
          af[i] = lds((as + (s / 4) * (BM * 128) + (16 * (i / 2) + (i % 2)) * 128) ^ (((2 * (s % 4)) ^ (i % 2)) * 16));
        } else {
          af[i] = lds((as + (i / 2) * 4096 + s * 512) ^ (((2 * (i % 2)) ^ (4 * (s % 2))) * 16));
        }
      }
#pragma unroll
      for (int j = 0; j < NJ; ++j) bf[j] = lds((bs + (j / 2) * 4096 + s * 512) ^ (((2 * (j % 2)) ^ (4 * (s % 2))) * 16));
#pragma unroll
      for (int i = 0; i < MI; ++i)
#pragma unroll
        for (int j = 0; j < NJ; ++j) dmma_m8n8k4(acc[i][j][0], acc[i][j][1], af[i], bf[j]);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(empty0 + 8 * stage);
  }

#pragma unroll
  for (int i = 0; i < MI; ++i) {
    const size_t row = size_t(row0) + c_row(i);
    if (row >= size_n) continue;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      // column-slots 2q, 2q+1 of tile j (same permutation as the B fragment)
      const size_t col = size_t(col0) + wc * (NJ * 8) + 16 * (j / 2) + 4 * (j % 2) + 2 * (q / 2) + 8 * (q % 2);
      if (col + 2 <= size_m) {
        double2 *dst = reinterpret_cast<double2 *>(C + row * size_m + col);
        if constexpr (ACC) {
          const double2 old = *dst;
          *dst = make_double2(__dadd_rn(old.x, acc[i][j][0]), __dadd_rn(old.y, acc[i][j][1]));
        } else {
          *dst = make_double2(acc[i][j][0], acc[i][j][1]);
        }
      }
    }
  }
}

template <bool TRANSPOSED_A, int BM>
__global__ void __launch_bounds__((TMA_WM * TMA_WN + 1) * 32, 1)
gemm_dmma_tma_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                     double *__restrict__ C, unsigned size_n, unsigned size_k, unsigned size_m, unsigned a_step,
                     unsigned b_step) {
  gemm_dmma_body<TRANSPOSED_A, BM, false>(map_a, map_b, C, size_n, size_k, size_m, a_step, b_step);
}

// C <- C + A * B (mm_kernel_enqueue_accumulate); instantiated in gemm_dmma_acc.cu only.
template <bool TRANSPOSED_A, int BM>
__global__ void __launch_bounds__((TMA_WM * TMA_WN + 1) * 32, 1)
gemm_dmma_accumulate_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                            double *__restrict__ C, unsigned size_n, unsigned size_k, unsigned size_m, unsigned a_step,
                            unsigned b_step) {
  gemm_dmma_body<TRANSPOSED_A, BM, true>(map_a, map_b, C, size_n, size_k, size_m, a_step, b_step);
}

template <bool TRANSPOSED_A, int BM, bool ACC>
constexpr auto dmma_kernel_ptr() {
  if constexpr (ACC) return gemm_dmma_accumulate_kernel<TRANSPOSED_A, BM>;
  else return gemm_dmma_tma_kernel<TRANSPOSED_A, BM>;
}

template <int BM, bool ACC>
int launch_dmma_tma(const GemmArgs &g) {
  const bool ta = (g.flags & MM_FLAG_TRANSPOSED_A) != 0;
  constexpr size_t SMEM = size_t(STAGES) * (BM * BK + BK * BN) * 8 + 2 * STAGES * 8 + 1024;
  constexpr int THREADS = (TMA_WM * TMA_WN + 1) * 32;
  MM_CUDA_TRY(cudaFuncSetAttribute(dmma_kernel_ptr<false, BM, ACC>(), cudaFuncAttributeMaxDynamicSharedMemorySize, int(SMEM)));
  MM_CUDA_TRY(cudaFuncSetAttribute(dmma_kernel_ptr<true, BM, ACC>(), cudaFuncAttributeMaxDynamicSharedMemorySize, int(SMEM)));
  if (g.dry_run) return MM_OK;
  CUtensorMap map_a, map_b;
  const unsigned na = g.batch.a_copies(), nb = g.batch.b_copies();
  const int ra = ta ? encode_sw128_3d_f64(&map_a, g.a, g.k, g.n, na, BK)
                    : encode_sw128_2d_f64(&map_a, g.a, uint64_t(na) * g.n, g.k, BM);
  const int rb = encode_sw128_3d_f64(&map_b, g.b, g.k, g.m, nb, BK);
  if (ra != 0 || rb != 0) return fail(MM_ERR_CUDA, "cuTensorMapEncodeTiled failed for the f64 operands");
  dim3 grid(ceil_div(g.m, BN), ceil_div(g.n, BM), g.batch.count);
  double *c = static_cast<double *>(g.c);
  const unsigned a_step = g.batch.shared_a ? 0u : 1u, b_step = g.batch.shared_b ? 0u : 1u;
  if (ta) {
    dmma_kernel_ptr<true, BM, ACC>()<<<grid, THREADS, SMEM, g.stream>>>(map_a, map_b, c, g.n, g.k, g.m, a_step, b_step);
  } else {
    dmma_kernel_ptr<false, BM, ACC>()<<<grid, THREADS, SMEM, g.stream>>>(map_a, map_b, c, g.n, g.k, g.m, a_step, b_step);
  }
  MM_CUDA_TRY(cudaGetLastError());
  return MM_OK;
}

// The launcher of both kernels; ACC selects the accumulate ones.
template <bool ACC>
int launch_dmma_impl(const GemmArgs &g) {
  const bool ta = (g.flags & MM_FLAG_TRANSPOSED_A) != 0;
  if (ta && (g.n % 2 != 0)) return fail(MM_ERR_UNSUPPORTED, "dmma path with transposed A needs even N");
  if (reinterpret_cast<uintptr_t>(g.a) % 16 != 0 || reinterpret_cast<uintptr_t>(g.b) % 16 != 0 ||
      reinterpret_cast<uintptr_t>(g.c) % 16 != 0) {
    return fail(MM_ERR_INVALID, "dmma path needs 16-byte aligned operands");
  }
  if (!get_encode_fn()) return fail(MM_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  // Tile height: 128 rows per CTA, or 64 when the 128-row tiling leaves the last wave mostly empty
  // (e.g. a 640-row block of 8192 columns: 320 tiles on 132 SMs = 2.42 waves; 640 half-height tiles
  // = 4.85 waves of half the duration).  The half-height tile reads B twice as
  // often per output row and runs ~2 % below the full tile, so it has to win by more than 5 %.
  // The tuning knob MM_TUNE_DMMA_TILE_ROWS (64 | 128) forces one of them.
  int sms = 132, dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  // (tiles of the whole batch: its problems run side by side in one grid)
  const double tiles_c = double(g.batch.count) * ceil_div(g.m, BN);
  const double t128 = double(ceil_div(g.n, 128)) * tiles_c, t64 = double(ceil_div(g.n, 64)) * tiles_c;
  const double cost128 = std::ceil(t128 / sms), cost64 = 0.5 * 1.05 * std::ceil(t64 / sms);
  const int forced = g.tuning ? g.tuning->dmma_tile_rows() : 0;
  const bool use64 = forced == 64 || (forced != 128 && cost64 < cost128);
  return use64 ? launch_dmma_tma<64, ACC>(g) : launch_dmma_tma<128, ACC>(g);
}

}  // namespace
}  // namespace mm
