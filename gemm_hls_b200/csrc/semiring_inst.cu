// One (data type, map operator) slice of the CUDA-core semiring tile kernel: the five reduce
// operators.  Compiled 30 times by gemm_hls_b200/build.py / CMakeLists.txt with
//   -DMM_INST_T=<C type> -DMM_INST_MAP=<MM_OP_* value>
#include "semiring_kernel.cuh"

#ifndef MM_INST_T
#error "compile with -DMM_INST_T=<type> -DMM_INST_MAP=<op>"
#endif

namespace mm {
using InstT = MM_INST_T;
MM_INSTANTIATE_SEMIRING(SemiringProduct, InstT, MM_INST_MAP,
                        MM_OP_MULTIPLY, MM_OP_ADD, MM_OP_MIN, MM_OP_MAX, MM_OP_AND)
}  // namespace mm
