// Accumulate instantiations of the wgmma GEMM (gemm_wgmma.cuh) for mm_kernel_enqueue_accumulate: C <- C + P, where
// P is what the plain kernel stores (the product rounded to the type of C) and the add is one IEEE add in that type
// (integer add modulo 256 for uint8_t), applied in the epilogue to the old C loaded at the addresses about to be
// stored.  {tf32, f16, bf16, u8} x {1, 2 CTAs} x {128, 256 columns}.  The plain kernels stay in gemm_tcgen05.cu and
// gemm_wgmma_bf16.cu, unchanged.
#include <cuda_bf16.h>

#include "gemm_wgmma.cuh"

namespace mm {

int wgmma_accumulate_gemm(int dtype, const void *a_op, const void *b_op, void *c, unsigned rows, unsigned k, unsigned m,
                          const Tuning &t, unsigned int *tile_sync, bool attributes_only, cudaStream_t stream,
                          const GemmBatch &batch, const HalfOperands &half) {
  CUtensorMap maps[5];
  LaunchPlan plan;
  const int rc = plan_gemm(dtype, a_op, b_op, c, rows, k, m, t, tile_sync, attributes_only, stream, batch, half, maps,
                           &plan);
  if (rc != MM_OK) return rc;
  const int cg = t.cta_group(), bn = t.block_n();
  switch (dtype) {
    case MM_DTYPE_FLOAT: return dispatch_variant<ptx::KIND_TF32, float, true>(cg, bn, plan);
    case MM_DTYPE_HALF: return dispatch_variant<ptx::KIND_F16, __half, true>(cg, bn, plan);
    case MM_DTYPE_BFLOAT16: return dispatch_variant<ptx::KIND_BF16, __nv_bfloat16, true>(cg, bn, plan);
    case MM_DTYPE_UINT8: return dispatch_variant<ptx::KIND_I8, unsigned char, true>(cg, bn, plan);
  }
  return fail(MM_ERR_UNSUPPORTED, "the wgmma path handles float, half, bfloat16 and uint8_t only");
}

}  // namespace mm
