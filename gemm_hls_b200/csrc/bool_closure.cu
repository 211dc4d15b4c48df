// Transitive closure of bit-packed Boolean matrices in place (mm_kernel_enqueue_bool_closure), by blocked
// Floyd–Warshall with blocks of B = 256 indices (DESIGN.md 3.10).  Round r, with K_r = [256 r, 256 r + w):
//   1. closure_diagonal_kernel: Warshall's bitset algorithm on D[K_r][K_r] in shared memory, one CTA per problem;
//   2. closure_tile_kernel over the row panel D[K_r][J] and the column panel D[I][K_r], I, J != K_r;
//   3. closure_tile_kernel over D[I][J], I, J != K_r.
// Phases 2 and 3 are the same update of one 256 x 256 tile, D[I][J] |= D[I][K_r] . D[K_r][J] (Boolean product, K =
// 256 bits): four b1 wgmma m64n256k256.  Each CTA owns its tile whole, and every operand it reads is either its own
// tile, read entirely before it writes, or a block no CTA of the launch writes.
#include "gemm_wgmma.cuh"

namespace mm {
namespace {

constexpr uint32_t CB = 256;                   // block of indices = tile side
constexpr uint32_t CT_A_BYTES = 64 * 128;      // A: 256 rows x 32 bytes as 64 rows x 128 B (row x at K slot x / 64)
constexpr uint32_t CT_B_BYTES = 256 * 128;     // B^T: 256 rows x 32 bytes at K slot 0 of 128-byte rows
constexpr size_t CT_SMEM = CT_A_BYTES + CT_B_BYTES + 1024;

// Byte offset of 16-byte chunk c (0..7) of row x in a 128-byte-swizzled K-major tile (what ptx::make_smem_desc_k_sw128
// describes): chunk position c XOR (x mod 8).
__device__ __forceinline__ uint32_t sw128(uint32_t x, uint32_t c) { return x * 128u + ((c ^ (x & 7u)) << 4); }

// Phase 1.  Thread i holds row i of the diagonal block (w <= 256 bits) in registers.  Step k ORs row k into every row
// with bit k set; row k does not change in step k, and its thread publishes it to shared memory at the end of step
// k - 1, so one barrier per step suffices.
__global__ void __launch_bounds__(CB) closure_diagonal_kernel(unsigned char *d, uint32_t n, uint32_t r) {
  __shared__ uint4 s_rows[CB][2];
  const uint32_t w = min(CB, n - r * CB);
  const size_t pitch = n / 8;
  unsigned char *blk = d + size_t(blockIdx.x) * n * pitch + size_t(r) * CB * pitch + r * (CB / 8);
  const uint32_t i = threadIdx.x;
  uint4 row[2] = {make_uint4(0, 0, 0, 0), make_uint4(0, 0, 0, 0)};
  if (i < w) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (h * 128u < w) row[h] = *reinterpret_cast<const uint4 *>(blk + i * pitch + 16 * h);
    }
  }
  s_rows[i][0] = row[0];
  s_rows[i][1] = row[1];
  __syncthreads();
#pragma unroll
  for (uint32_t kw = 0; kw < CB / 32; ++kw) {
    if (kw * 32 >= w) break;
    const uint4 &hw = row[kw / 4];
    for (uint32_t kb = 0; kb < 32; ++kb) {
      const uint32_t k = kw * 32 + kb;
      const uint32_t mine = (kw % 4 == 0) ? hw.x : (kw % 4 == 1) ? hw.y : (kw % 4 == 2) ? hw.z : hw.w;
      const uint4 a = s_rows[k][0], b = s_rows[k][1];
      if ((mine >> kb) & 1u) {
        row[0].x |= a.x; row[0].y |= a.y; row[0].z |= a.z; row[0].w |= a.w;
        row[1].x |= b.x; row[1].y |= b.y; row[1].z |= b.z; row[1].w |= b.w;
      }
      if (i == k + 1) {
        s_rows[i][0] = row[0];
        s_rows[i][1] = row[1];
      }
      __syncthreads();
    }
  }
  if (i < w) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (h * 128u < w) *reinterpret_cast<uint4 *>(blk + i * pitch + 16 * h) = row[h];
    }
  }
}

// Phases 2 (PANELS) and 3: one 256 x 256 tile (bi, bj) of problem blockIdx.y per CTA, one warpgroup.  Two
// instantiations of one body, so that profiles tell the phases apart.
template <bool PANELS>
__global__ void __launch_bounds__(128, 3) closure_tile_kernel(unsigned char *d, uint32_t n, uint32_t r) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  const uint32_t sa = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sb = sa + CT_A_BYTES;
  const uint32_t nb = (n + CB - 1) / CB, o = nb - 1;
  uint32_t bi, bj;
  const uint32_t t = blockIdx.x;
  if (PANELS) {
    if (t < o) { bi = r; bj = t + (t >= r ? 1u : 0u); }
    else { bi = (t - o) + (t - o >= r ? 1u : 0u); bj = r; }
  } else {
    bi = t / o; bj = t % o;
    bi += bi >= r ? 1u : 0u;
    bj += bj >= r ? 1u : 0u;
  }
  const size_t pitch = n / 8;
  unsigned char *D = d + size_t(blockIdx.y) * n * pitch;
  const uint32_t i0 = bi * CB, j0 = bj * CB, k0 = r * CB;
  const uint32_t tid = threadIdx.x, warp = tid / 32, lane = tid % 32;
  const uint32_t r_in = lane / 4, q = lane % 4;
  // The global loads are issued before their values are needed: A = D[I][K_r] and B = D[K_r][J] (thread tid holds
  // rows tid and 128 + tid of both) and the old words of D[I][J] that this lane updates in the first slab, all at
  // once; the old words of slab s + 1 while slab s computes.  Slab s: row 16 warp + r_in + 8 (q / 2) of rows
  // 64 s .. + 64, columns 128 (q % 2) .. + 128.  Indices past n read as zero: N is a multiple of 128, so each 16-byte
  // chunk is wholly inside D or outside.
  uint4 av[2][2], bv[2][2];
#pragma unroll
  for (uint32_t half = 0; half < 2; ++half) {
    const uint32_t x = tid + 128u * half;
#pragma unroll
    for (uint32_t h = 0; h < 2; ++h) {
      av[half][h] = bv[half][h] = make_uint4(0, 0, 0, 0);
      if (i0 + x < n && k0 + 128 * h < n) {
        av[half][h] = *reinterpret_cast<const uint4 *>(D + size_t(i0 + x) * pitch + k0 / 8 + 16 * h);
      }
      if (k0 + x < n && j0 + 128 * h < n) {
        bv[half][h] = *reinterpret_cast<const uint4 *>(D + size_t(k0 + x) * pitch + j0 / 8 + 16 * h);
      }
    }
  }
  const uint32_t c_col = j0 + 128 * (q % 2);
  auto old_words = [&](uint32_t s) {
    const uint32_t row = i0 + 64 * s + 16 * warp + r_in + 8 * (q / 2);
    uint4 v = make_uint4(0, 0, 0, 0);
    if (row < n && c_col < n) v = *reinterpret_cast<const uint4 *>(D + size_t(row) * pitch + c_col / 8);
    return v;
  };
  uint4 old = old_words(0);
  // A: row x of the tile into K slot x / 64 of row x % 64.  B: warp w holds k rows 32 w + lane and 128 + 32 w + lane,
  // whose 32 x 32 blocks it transposes into rows j of B^T.
#pragma unroll
  for (uint32_t half = 0; half < 2; ++half) {
    const uint32_t x = tid + 128u * half;
#pragma unroll
    for (uint32_t h = 0; h < 2; ++h) {
      const uint4 &v = av[half][h];
      ptx::st_shared_v4(sa + sw128(x % 64, 2 * (x / 64) + h), v.x, v.y, v.z, v.w);
    }
    const uint32_t bw[8] = {bv[half][0].x, bv[half][0].y, bv[half][0].z, bv[half][0].w,
                            bv[half][1].x, bv[half][1].y, bv[half][1].z, bv[half][1].w};
    const uint32_t kg = x / 32;  // k word of the transposed rows
#pragma unroll
    for (uint32_t mg = 0; mg < 8; ++mg) {
      const uint32_t j = 32 * mg + lane;
      const uint32_t y = warp_transpose32(bw[mg], lane);
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(sb + sw128(j, kg / 4) + 4 * (kg % 4)), "r"(y) : "memory");
    }
  }
  ptx::fence_proxy_async_smem();  // generic-proxy writes -> the wgmma's reads
  __syncthreads();

  const uint64_t adesc = ptx::make_smem_desc_k_sw128(sa), bdesc = ptx::make_smem_desc_k_sw128(sb);
  uint32_t acc[128];
#pragma unroll
  for (uint32_t s = 0; s < 4; ++s) {
    ptx::wgmma_fence();
    ptx::wgmma<ptx::KIND_B1, 256>(acc, adesc + uint64_t(2 * s), bdesc, 0u);
    ptx::wgmma_commit();
    const uint4 next = s < 3 ? old_words(s + 1) : make_uint4(0, 0, 0, 0);
    ptx::wgmma_wait<0>();
    uint32_t w[2][8];
    pack_bit_words<256>(acc, q, w);
    const uint32_t row = i0 + 64 * s + 16 * warp + r_in + 8 * (q / 2);
#pragma unroll
    for (uint32_t i = 0; i < 2; ++i) {
#pragma unroll
      for (uint32_t g = 0; g < 2; ++g) {
        if (q == 2 * i + g && row < n && c_col < n) {
          *reinterpret_cast<uint4 *>(D + size_t(row) * pitch + c_col / 8) = make_uint4(
              old.x | w[i][4 * g], old.y | w[i][4 * g + 1], old.z | w[i][4 * g + 2], old.w | w[i][4 * g + 3]);
        }
      }
    }
    old = next;
  }
}

}  // namespace

int bool_closure(void *d, unsigned n, unsigned batch, cudaStream_t stream) {
  unsigned char *dp = static_cast<unsigned char *>(d);
  const uint32_t nb = ceil_div(n, CB);
  // also loads both kernels before a first launch, which may be inside a stream capture
  const cudaFuncAttribute smem_attr = cudaFuncAttributeMaxDynamicSharedMemorySize;
  MM_CUDA_TRY(cudaFuncSetAttribute(closure_tile_kernel<true>, smem_attr, int(CT_SMEM)));
  MM_CUDA_TRY(cudaFuncSetAttribute(closure_tile_kernel<false>, smem_attr, int(CT_SMEM)));
  MM_CUDA_TRY(cudaFuncSetAttribute(closure_diagonal_kernel, smem_attr, 0));
  for (uint32_t r = 0; r < nb; ++r) {
    closure_diagonal_kernel<<<batch, CB, 0, stream>>>(dp, n, r);
    MM_CUDA_TRY(cudaGetLastError());
    if (nb == 1) break;
    closure_tile_kernel<true><<<dim3(2 * (nb - 1), batch), 128, CT_SMEM, stream>>>(dp, n, r);
    MM_CUDA_TRY(cudaGetLastError());
    closure_tile_kernel<false><<<dim3((nb - 1) * (nb - 1), batch), 128, CT_SMEM, stream>>>(dp, n, r);
    MM_CUDA_TRY(cudaGetLastError());
  }
  return MM_OK;
}

}  // namespace mm
