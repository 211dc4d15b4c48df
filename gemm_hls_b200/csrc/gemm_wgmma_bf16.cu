// bf16 instantiations of the wgmma GEMM (gemm_wgmma.cuh): (Multiply, Add) on bfloat16 operands with FP32
// accumulation and one rounding to bfloat16 per element of C (cvt.rn.bf16x2.f32 in the epilogue).  Same
// descriptors, swizzle and shared-memory geometry as f16; {1, 2 CTAs} x {128, 256 columns}.  Operand
// preparation is gemm_tcgen05.cu's: bf16 and half move the same bits.
#include <cuda_bf16.h>

#include "gemm_wgmma.cuh"

namespace mm {

int wgmma_bf16_gemm(const void *a_op, const void *b_op, void *c, unsigned rows, unsigned k, unsigned m, const Tuning &t,
                    unsigned int *tile_sync, bool attributes_only, cudaStream_t stream, const GemmBatch &batch) {
  CUtensorMap maps[5];
  LaunchPlan plan;
  const int rc = plan_gemm(MM_DTYPE_BFLOAT16, a_op, b_op, c, rows, k, m, t, tile_sync, attributes_only, stream, batch,
                           HalfOperands{}, maps, &plan);
  if (rc != MM_OK) return rc;
  return dispatch_variant<ptx::KIND_BF16, __nv_bfloat16>(t.cta_group(), t.block_n(), plan);
}

}  // namespace mm
