// Bit-packed Boolean product (mm_kernel_enqueue_bool): C[i][j] = OR_k A[i][k] AND B[k][j] on the b1 tensor cores.
// The wgmma GEMM (gemm_wgmma.cuh) instantiated with KIND_B1: wgmma m64nNk256.s32.b1.b1.and.popc counts the k with
// a AND b over 256 bits of K, and the epilogue stores count > 0 as one bit (store_bit_tile).  Both operands are
// moved as bytes, with the descriptors, swizzle and ring of the u8 path: a K-major row of K bits is K / 8 bytes.
// B arrives row-major K x M, so bit_transpose_kernel first writes its K-major M x K copy into the context's scratch.
// {1, 2 CTAs} x {128, 256 columns}.
#include "gemm_wgmma.cuh"

namespace mm {
namespace {

constexpr int BT_TILE = 256;  // bits per side of the tile one CTA of bit_transpose_kernel moves
constexpr int BT_WORDS = BT_TILE / 32;

// `copies` packed K x M bit matrices (rows of M / 8 bytes) at `b` -> their M x K transposes (rows of K / 8 bytes) at
// `bt`.  One CTA per 256 x 256 tile: coalesced 32-byte row segments into shared memory, eight warps transposing
// 32 x 32 blocks with warp_transpose32, 32-byte row segments out.  K and M are multiples of 128, so a 128-bit word is
// wholly inside the matrix or wholly outside.
__global__ void __launch_bounds__(256) bit_transpose_kernel(const uint32_t *__restrict__ b, uint32_t *__restrict__ bt,
                                                             uint32_t k, uint32_t m) {
  __shared__ uint32_t s_in[BT_TILE][BT_WORDS + 1];   // [k row][m word]; +1: conflict-free column reads
  __shared__ uint32_t s_out[BT_TILE][BT_WORDS + 1];  // [m row][k word]
  const uint32_t mw = m / 32, kw = k / 32;           // words per row of B and of its transpose
  const uint32_t tiles_m = (m + BT_TILE - 1) / BT_TILE, tiles_k = (k + BT_TILE - 1) / BT_TILE;
  const size_t prob = blockIdx.z;
  const uint32_t *src = b + prob * k * mw;
  uint32_t *dst = bt + prob * m * kw;
  const uint32_t warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const uint32_t r = threadIdx.x;  // this thread's row of the tile, on the way in and on the way out
  for (uint32_t t = blockIdx.x; t < tiles_m * tiles_k; t += gridDim.x) {
    const uint32_t m0 = (t % tiles_m) * BT_TILE, k0 = (t / tiles_m) * BT_TILE;
    // row k0 + r, words m0 / 32 .. + 8 (zeros outside the matrix)
    uint4 v[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t w0 = m0 / 32 + 4 * h;
      v[h] = make_uint4(0, 0, 0, 0);
      if (k0 + r < k && w0 < mw) v[h] = *reinterpret_cast<const uint4 *>(src + size_t(k0 + r) * mw + w0);
    }
    __syncthreads();  // the previous tile's s_out has been written out
    s_in[r][0] = v[0].x; s_in[r][1] = v[0].y; s_in[r][2] = v[0].z; s_in[r][3] = v[0].w;
    s_in[r][4] = v[1].x; s_in[r][5] = v[1].y; s_in[r][6] = v[1].z; s_in[r][7] = v[1].w;
    __syncthreads();
    // 64 blocks of 32 x 32: block (kg, mg) = k rows 32 kg.., m word mg
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const uint32_t blk = warp * 8 + i, kg = blk / BT_WORDS, mg = blk % BT_WORDS;
      s_out[32 * mg + lane][kg] = warp_transpose32(s_in[32 * kg + lane][mg], lane);
    }
    __syncthreads();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t w0 = k0 / 32 + 4 * h;
      if (m0 + r < m && w0 < kw) {
        *reinterpret_cast<uint4 *>(dst + size_t(m0 + r) * kw + w0) =
            make_uint4(s_out[r][4 * h], s_out[r][4 * h + 1], s_out[r][4 * h + 2], s_out[r][4 * h + 3]);
      }
    }
  }
}

// C (`batch` packed rows x cols bit matrices, rows of cols / 8 bytes) for store_bit_tile's TMA stores: boxes of
// 16 rows x BN / 8 bytes, unswizzled, three dimensions so that a partial last row block is clipped per problem.
int make_bit_c_map(CUtensorMap *map, void *base, uint64_t rows, uint64_t cols, uint64_t batch, uint32_t bn) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return fail(MM_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t gdim[3] = {cols / 8, rows, batch};
  cuuint64_t gstride[2] = {cols / 8, rows * cols / 8};
  cuuint32_t box[3] = {bn / 8, EPI_ROWS, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, base, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    return fail(MM_ERR_CUDA, "cuTensorMapEncodeTiled (bit C) failed with CUresult " + std::to_string(int(r)));
  }
  return MM_OK;
}

}  // namespace

int bool_transpose_b(const void *b, void *bt, unsigned k, unsigned m, unsigned batch, cudaStream_t stream) {
  const uint32_t tiles = ceil_div(m, BT_TILE) * ceil_div(k, BT_TILE);
  const uint32_t grid = std::min<uint32_t>(tiles, uint32_t(num_sms()) * 8);
  bit_transpose_kernel<<<dim3(grid, 1, batch), 256, 0, stream>>>(static_cast<const uint32_t *>(b),
                                                                  static_cast<uint32_t *>(bt), k, m);
  MM_CUDA_TRY(cudaGetLastError());
  return MM_OK;
}

int bool_gemm(const void *a, const void *bt, void *c, unsigned n, unsigned k, unsigned m, unsigned batch,
              const Tuning &t, unsigned int *tile_sync, cudaStream_t stream) {
  // byte operands of k / 8 bytes per row; the u8 C map plan_gemm would make is replaced by the bit one
  Tuning tb = t;
  tb.v[MM_TUNE_TCGEN05_TMA_STORE] = 0;
  CUtensorMap maps[5];
  LaunchPlan plan;
  GemmBatch bt_batch;
  bt_batch.count = batch;
  int rc = plan_gemm(MM_DTYPE_UINT8, a, bt, c, n, k / 8, m, tb, tile_sync, false, stream, bt_batch, HalfOperands{},
                     maps, &plan);
  if (rc != MM_OK) return rc;
  if (t.tma_store()) {
    if ((rc = make_bit_c_map(&maps[2], c, n, m, batch, uint32_t(t.block_n()))) != MM_OK) return rc;
    plan.p.tma_store = 1u;
  }
  return dispatch_variant<ptx::KIND_B1, unsigned char>(t.cta_group(), t.block_n(), plan);
}

}  // namespace mm
