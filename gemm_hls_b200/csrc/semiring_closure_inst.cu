// One (data type, map operator) slice of the closure kernels: the Min / Max reduces (and FMNMX for float).
// Compiled once per (type, map) by gemm_hls_b200/build.py / CMakeLists.txt with
//   -DMM_INST_T=<C type> -DMM_INST_MAP=<MM_OP_* value>
#include "semiring_closure_kernel.cuh"

#ifndef MM_INST_T
#error "compile with -DMM_INST_T=<type> -DMM_INST_MAP=<op>"
#endif

namespace mm {
using InstT = MM_INST_T;
MM_INSTANTIATE_SEMIRING(SemiringClosure, InstT, MM_INST_MAP, MM_OP_MIN, MM_OP_MAX)
}  // namespace mm
