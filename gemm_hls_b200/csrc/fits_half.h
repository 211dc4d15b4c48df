// Whether a TF32-rounded float is exactly a normal half (or zero): the test that lets the float GEMM run a problem on
// the f16 wgmma.  Plain C++ as well as CUDA, so that tests/test_fits_half_cpu.py can compile it with g++ and check it
// against numpy on every TF32 bit pattern.
#pragma once

#include <cstdint>

#ifdef __CUDACC__
#define MM_HOST_DEVICE __host__ __device__
#else
#define MM_HOST_DEVICE
#endif

namespace mm {

// `bits`: a float rounded to nearest TF32 (10 mantissa bits, the low 13 bits zero).  A half has the same 10 mantissa
// bits, so the value is a half exactly when its exponent fits: v == +-0 or 2^-14 <= |v| < 2^16 (biased float exponent
// 113 .. 142).  Infinities, NaN, float subnormals and the half-subnormal band below 2^-14 do not fit.
MM_HOST_DEVICE constexpr bool tf32_fits_half(uint32_t bits) {
  return (bits & 0x7FFFFFFFu) == 0u || ((bits >> 23) & 0xFFu) - 113u < 30u;
}

}  // namespace mm
