// Semiring functors for the device kernels: same interface as the reference's hlslib::op
// functors (hlslib/include/hlslib/xilinx/Operators.h:20-100) — `static T Apply(a, b)` and
// `static constexpr T identity()` — so a (Map, Reduce) pair plugs into the kernels exactly like
// MM_MAP_OP / MM_REDUCE_OP plug into the reference's ProcessingElement (kernel/Compute.cpp:129-133).
//
// Rounding contract: Apply() performs ONE correctly rounded operation in T (no FMA contraction
// across Map and Reduce), so a kernel that reduces sequentially over k reproduces the
// reference's Naive<> (include/Utility.h:18-42) bit for bit.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <cfloat>
#include <climits>
#include <cstdint>

#include "../../include/mm_b200.h"

namespace mm {

// ---- per-type primitives ---------------------------------------------------------------------
template <typename T>
struct Prim {
  static __host__ __device__ __forceinline__ T add(T a, T b) { return static_cast<T>(a + b); }
  static __host__ __device__ __forceinline__ T mul(T a, T b) { return static_cast<T>(a * b); }
  static __host__ __device__ __forceinline__ bool lt(T a, T b) { return a < b; }
  static __host__ __device__ __forceinline__ bool nz(T a) { return a != T(0); }
  static __host__ __device__ __forceinline__ T zero() { return T(0); }
  static __host__ __device__ __forceinline__ T one() { return T(1); }
};

template <>
struct Prim<float> {
  // __fadd_rn/__fmul_rn are never contracted into an FMA by the compiler.
  static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
  static __device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
  static __device__ __forceinline__ bool lt(float a, float b) { return a < b; }
  static __device__ __forceinline__ bool nz(float a) { return a != 0.0f; }
  static __device__ __forceinline__ float zero() { return 0.0f; }
  static __device__ __forceinline__ float one() { return 1.0f; }
  // numeric_limits<float>::max() / ::min()
  static __device__ __forceinline__ float max_value() { return FLT_MAX; }
  static __device__ __forceinline__ float min_value() { return FLT_MIN; }
};

template <>
struct Prim<double> {
  static __device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
  static __device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
  static __device__ __forceinline__ bool lt(double a, double b) { return a < b; }
  static __device__ __forceinline__ bool nz(double a) { return a != 0.0; }
  static __device__ __forceinline__ double zero() { return 0.0; }
  static __device__ __forceinline__ double one() { return 1.0; }
  static __device__ __forceinline__ double max_value() { return DBL_MAX; }
  static __device__ __forceinline__ double min_value() { return DBL_MIN; }
};

template <>
struct Prim<__half> {
  static __device__ __forceinline__ __half add(__half a, __half b) { return __hadd_rn(a, b); }
  static __device__ __forceinline__ __half mul(__half a, __half b) { return __hmul_rn(a, b); }
  static __device__ __forceinline__ bool lt(__half a, __half b) { return __hlt(a, b); }
  static __device__ __forceinline__ bool nz(__half a) { return __hneu(a, __ushort_as_half(0)); }  // `a != 0`: true for NaN
  static __device__ __forceinline__ __half zero() { return __ushort_as_half(0x0000); }
  static __device__ __forceinline__ __half one() { return __ushort_as_half(0x3C00); }
  static __device__ __forceinline__ __half max_value() { return __ushort_as_half(0x7BFF); }  // 65504
  static __device__ __forceinline__ __half min_value() { return __ushort_as_half(0x0400); }  // 2^-14
};

template <>
struct Prim<__nv_bfloat16> {
  static __device__ __forceinline__ __nv_bfloat16 add(__nv_bfloat16 a, __nv_bfloat16 b) { return __hadd_rn(a, b); }
  static __device__ __forceinline__ __nv_bfloat16 mul(__nv_bfloat16 a, __nv_bfloat16 b) { return __hmul_rn(a, b); }
  static __device__ __forceinline__ bool lt(__nv_bfloat16 a, __nv_bfloat16 b) { return __hlt(a, b); }
  static __device__ __forceinline__ bool nz(__nv_bfloat16 a) { return __hneu(a, __ushort_as_bfloat16(0)); }  // true for NaN
  static __device__ __forceinline__ __nv_bfloat16 zero() { return __ushort_as_bfloat16(0x0000); }
  static __device__ __forceinline__ __nv_bfloat16 one() { return __ushort_as_bfloat16(0x3F80); }
  static __device__ __forceinline__ __nv_bfloat16 max_value() { return __ushort_as_bfloat16(0x7F7F); }  // 0x1.fep127
  static __device__ __forceinline__ __nv_bfloat16 min_value() { return __ushort_as_bfloat16(0x0080); }  // 2^-126
};

template <typename T>
struct IntLimits;
template <>
struct IntLimits<int> {
  static __host__ __device__ __forceinline__ int max_value() { return INT_MAX; }
  static __host__ __device__ __forceinline__ int min_value() { return INT_MIN; }
};
template <>
struct IntLimits<unsigned> {
  static __host__ __device__ __forceinline__ unsigned max_value() { return UINT_MAX; }
  static __host__ __device__ __forceinline__ unsigned min_value() { return 0u; }
};
template <>
struct IntLimits<unsigned char> {
  static __host__ __device__ __forceinline__ unsigned char max_value() { return 255; }
  static __host__ __device__ __forceinline__ unsigned char min_value() { return 0; }
};

template <typename T>
struct Lim {
  static __device__ __forceinline__ T max_value() { return IntLimits<T>::max_value(); }
  static __device__ __forceinline__ T min_value() { return IntLimits<T>::min_value(); }
};
template <> struct Lim<float> : Prim<float> {};
template <> struct Lim<double> : Prim<double> {};
template <> struct Lim<__half> : Prim<__half> {};
template <> struct Lim<__nv_bfloat16> : Prim<__nv_bfloat16> {};

// ---- the functors (Operators.h) ---------------------------------------------------------------
template <typename T>
struct Sum {  // Operators.h:20-33
  static __device__ __forceinline__ T Apply(T a, T b) { return Prim<T>::add(a, b); }
  static __device__ __forceinline__ T identity() { return Prim<T>::zero(); }
};
template <typename T>
using Add = Sum<T>;  // Operators.h:35-36

template <typename T>
struct Product {  // Operators.h:45-58
  static __device__ __forceinline__ T Apply(T a, T b) { return Prim<T>::mul(a, b); }
  static __device__ __forceinline__ T identity() { return Prim<T>::one(); }
};
template <typename T>
using Multiply = Product<T>;  // Operators.h:60-61

template <typename T>
struct And {  // Operators.h:63-74 — `a && b` converted back to T
  static __device__ __forceinline__ T Apply(T a, T b) {
    return (Prim<T>::nz(a) && Prim<T>::nz(b)) ? Prim<T>::one() : Prim<T>::zero();
  }
  static __device__ __forceinline__ T identity() { return Prim<T>::one(); }
};

template <typename T>
struct Min {  // Operators.h:76-87
  static __device__ __forceinline__ T Apply(T a, T b) { return Prim<T>::lt(a, b) ? a : b; }
  static __device__ __forceinline__ T identity() { return Lim<T>::max_value(); }
};

template <typename T>
struct Max {  // Operators.h:89-100 — identity is numeric_limits<T>::min() as in the reference
  static __device__ __forceinline__ T Apply(T a, T b) { return Prim<T>::lt(b, a) ? a : b; }
  static __device__ __forceinline__ T identity() { return Lim<T>::min_value(); }
};

// Hardware min / max for float (FMNMX): one
// instruction instead of the compare + select that the literal `(a < b) ? a : b` needs.  Identical
// results for all finite inputs except the sign of a zero when the operands are -0 and +0, and
// NaNs are dropped instead of propagated; selected for float unless MM_FLAG_EXACT is given.
template <typename T>
struct MinFast : Min<T> {};
template <typename T>
struct MaxFast : Max<T> {};
template <>
struct MinFast<float> {
  static __device__ __forceinline__ float Apply(float a, float b) { return fminf(a, b); }
  static __device__ __forceinline__ float identity() { return Lim<float>::max_value(); }
};
template <>
struct MaxFast<float> {
  static __device__ __forceinline__ float Apply(float a, float b) { return fmaxf(a, b); }
  static __device__ __forceinline__ float identity() { return Lim<float>::min_value(); }
};

// ---- witnesses (mm_kernel_enqueue_witness) -------------------------------------------------------------
// Selects<Reduce>::apply(acc, t): whether the step acc <- Reduce(acc, t) keeps the new term t.  The literal
// `(acc < t) ? acc : t` keeps t unless acc is strictly better, so ties go to the later k and a NaN term is kept;
// FMNMX keeps t only when it is strictly better, so ties go to the earlier k and a NaN term is dropped.
template <class Reduce>
struct Selects;
template <typename T>
struct Selects<Min<T>> {
  static __device__ __forceinline__ bool apply(T acc, T t) { return !Prim<T>::lt(acc, t); }
};
template <typename T>
struct Selects<Max<T>> {
  static __device__ __forceinline__ bool apply(T acc, T t) { return !Prim<T>::lt(t, acc); }
};
template <typename T>
struct Selects<MinFast<T>> : Selects<Min<T>> {};
template <typename T>
struct Selects<MaxFast<T>> : Selects<Max<T>> {};
template <>
struct Selects<MinFast<float>> {
  static __device__ __forceinline__ bool apply(float acc, float t) { return t < acc; }
};
template <>
struct Selects<MaxFast<float>> {
  static __device__ __forceinline__ bool apply(float acc, float t) { return acc < t; }
};

// ---- packed pairs (half) -------------------------------------------------------------------------
// HADD2 / HMUL2 do two IEEE round-to-nearest half operations per instruction, each half rounded exactly like the
// scalar __hadd_rn / __hmul_rn; the _rn intrinsics are never contracted into an HFMA2 (a single rounding, which
// Naive<> does not do).  Used when BOTH Map and Reduce are Sum / Product — (Multiply, Add) under MM_FLAG_EXACT, the
// datapath the half host programs run by default — for two adjacent columns of C at a time.
template <class Op>
struct PackedOpH {
  static constexpr bool value = false;
};
template <>
struct PackedOpH<Sum<__half>> {
  static constexpr bool value = true;
  static __device__ __forceinline__ __half2 Apply2(__half2 a, __half2 b) { return __hadd2_rn(a, b); }
};
template <>
struct PackedOpH<Product<__half>> {
  static constexpr bool value = true;
  static __device__ __forceinline__ __half2 Apply2(__half2 a, __half2 b) { return __hmul2_rn(a, b); }
};

// bfloat16: the same with HADD2.BF16 / HMUL2.BF16 (__hadd2_rn / __hmul2_rn, never contracted into an HFMA2.BF16).
template <class Op>
struct PackedOpB {
  static constexpr bool value = false;
};
template <>
struct PackedOpB<Sum<__nv_bfloat16>> {
  static constexpr bool value = true;
  static __device__ __forceinline__ __nv_bfloat162 Apply2(__nv_bfloat162 a, __nv_bfloat162 b) { return __hadd2_rn(a, b); }
};
template <>
struct PackedOpB<Product<__nv_bfloat16>> {
  static constexpr bool value = true;
  static __device__ __forceinline__ __nv_bfloat162 Apply2(__nv_bfloat162 a, __nv_bfloat162 b) { return __hmul2_rn(a, b); }
};

// The pair type of a 2-byte floating-point T and its conversions: broadcast, (low, high) -> pair, pair -> low / high.
template <typename T>
struct Packed2 {
  using type = __half2;  // placeholder for the types without a packed path
};
template <>
struct Packed2<__half> {
  using type = __half2;
  static __device__ __forceinline__ __half2 bcast(__half x) { return __half2half2(x); }
  static __device__ __forceinline__ __half2 pair(__half lo, __half hi) { return __halves2half2(lo, hi); }
  static __device__ __forceinline__ __half lo(__half2 x) { return __low2half(x); }
  static __device__ __forceinline__ __half hi(__half2 x) { return __high2half(x); }
};
template <>
struct Packed2<__nv_bfloat16> {
  using type = __nv_bfloat162;
  static __device__ __forceinline__ __nv_bfloat162 bcast(__nv_bfloat16 x) { return __bfloat162bfloat162(x); }
  static __device__ __forceinline__ __nv_bfloat162 pair(__nv_bfloat16 lo, __nv_bfloat16 hi) { return __halves2bfloat162(lo, hi); }
  static __device__ __forceinline__ __nv_bfloat16 lo(__nv_bfloat162 x) { return __low2bfloat16(x); }
  static __device__ __forceinline__ __nv_bfloat16 hi(__nv_bfloat162 x) { return __high2bfloat16(x); }
};

// internal operator codes (never cross the C-ABI)
enum { MM_OP_MIN_FAST = 5, MM_OP_MAX_FAST = 6 };

template <typename T, int OP>
struct OpSelect;
template <typename T> struct OpSelect<T, MM_OP_MULTIPLY> { using type = Product<T>; };
template <typename T> struct OpSelect<T, MM_OP_ADD> { using type = Sum<T>; };
template <typename T> struct OpSelect<T, MM_OP_MIN> { using type = Min<T>; };
template <typename T> struct OpSelect<T, MM_OP_MAX> { using type = Max<T>; };
template <typename T> struct OpSelect<T, MM_OP_AND> { using type = And<T>; };
template <typename T> struct OpSelect<T, MM_OP_MIN_FAST> { using type = MinFast<T>; };
template <typename T> struct OpSelect<T, MM_OP_MAX_FAST> { using type = MaxFast<T>; };

// MM_DTYPE_* -> C type
template <int DTYPE> struct DTypeOf;
template <> struct DTypeOf<MM_DTYPE_HALF> { using type = __half; };
template <> struct DTypeOf<MM_DTYPE_FLOAT> { using type = float; };
template <> struct DTypeOf<MM_DTYPE_DOUBLE> { using type = double; };
template <> struct DTypeOf<MM_DTYPE_INT32> { using type = int; };
template <> struct DTypeOf<MM_DTYPE_UINT32> { using type = unsigned; };
template <> struct DTypeOf<MM_DTYPE_UINT8> { using type = unsigned char; };
template <> struct DTypeOf<MM_DTYPE_BFLOAT16> { using type = __nv_bfloat16; };

}  // namespace mm
