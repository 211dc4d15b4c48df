// The accumulate DMMA GEMM for double (mm_kernel_enqueue_accumulate): C <- C + A * B, the product computed exactly as
// gemm_dmma.cu computes it and added to C's old value by one __dadd_rn per element in the epilogue.
// {row-major A, A stored K x N} x {128, 64 rows}.  Kernel and launcher in gemm_dmma.cuh.
#include "gemm_dmma.cuh"

namespace mm {

int launch_dmma_accumulate(const GemmArgs &g) { return launch_dmma_impl<true>(g); }

}  // namespace mm
