// The plain DMMA GEMM for double: C = A * B.  Kernel and launcher in gemm_dmma.cuh.
#include "gemm_dmma.cuh"

namespace mm {

int launch_dmma(const GemmArgs &g) { return launch_dmma_impl<false>(g); }

}  // namespace mm
