// Host-facing declarations of the hot path — counterpart of the reference's
// include/MatrixMultiplication.h (kSeed :14, memory widths :18-27, the extern "C" kernel
// prototype :155-171).  The reference's MemoryPack*_t arrays are bit-identical to flat Data_t
// arrays (include/Utility.h:44-63), so the GPU entry takes flat pointers.
#pragma once

#include "Config.h"

constexpr int kSeed = 5;  // include/MatrixMultiplication.h:14

constexpr int kMemoryWidthK = kMemoryWidthBytesK / sizeof(Data_t);  // :18
constexpr int kMemoryWidthM = kMemoryWidthBytesM / sizeof(Data_t);  // :24
static_assert(kMemoryWidthBytesK == 64 && kMemoryWidthBytesM == 64,
              "libmm_b200 implements the reference's default 64-byte memory word");

extern "C" {

// Same name, argument order and meaning as the reference's simulation entry
// (include/MatrixMultiplication.h:155-171; called with HOST pointers at
// test/TestSimulation.cpp:66).  Blocking: H2D copies, the sm_90a kernels, D2H copy of C.
// Throws std::runtime_error (what() = mm_last_error()) on failure.
#ifdef MM_DYNAMIC_SIZES
void MatrixMultiplicationKernel(Data_t const a[], Data_t const b[], Data_t c[], const unsigned size_n,
                                const unsigned size_k, const unsigned size_m);
#else
void MatrixMultiplicationKernel(Data_t const a[], Data_t const b[], Data_t c[]);
#endif
}
