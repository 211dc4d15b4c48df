// ORACLE — TEST INFRASTRUCTURE ONLY.
//
// CPU restatement of the reference's result definition for the hot path.  Only
// tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
// reference legs may load this; the product library (libmm_b200.so) never does.
//
// What is restated (reference file:line, all in the reference checkout):
//   * Naive<OperatorMap, OperatorReduce>        include/Utility.h:18-42
//       acc = OperatorReduce::identity(); for k: acc = Reduce(acc, Map(a, b));
//       row-major A (N x K; K x N iff MM_TRANSPOSED_A, Utility.h:31-35),
//       row-major B (K x M), row-major C (N x M); accumulation type == Data_t.
//   * the semiring functors and their identities hlslib/include/hlslib/xilinx/Operators.h:20-100
//       Sum/Add 0, Product/Multiply 1, And true, Min numeric_limits<T>::max(),
//       Max numeric_limits<T>::min()  (sic: smallest POSITIVE value for fp).
//   * the input recipe                          test/TestSimulation.cpp:42-55,
//       host/RunHardware.cpp:31-35,99-104, include/MatrixMultiplication.h:14
//       std::default_random_engine(kSeed = 5); uniform_real_distribution<double>(1, 10)
//       (uniform_int_distribution<unsigned long>(1, 10) for integral Data_t);
//       ALL of A is drawn first, then all of B; each draw is cast to Data_t.
//   * the acceptance criterion                  test/TestSimulation.cpp:75-92,
//       host/RunHardware.cpp:207-224
//       floating point: mismatch iff |test - ref| / ref > 1e-3 (computed in
//       Data_t; a NaN quotient is NOT a mismatch); integral: mismatch iff != .
//
// Pinning: oracle/build.py compiles the reference's own Naive<> in place into
// oracle/_ref/ and tests/test_oracle.py asserts bit-equality of this
// restatement against it and against tests/golden/*.json.  `half` is the one
// exception: the reference's half is Xilinx' hls_half.h, which is not vendored,
// so half parity is UNPINNED at the bit level (see oracle/README.md).
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <limits>
#include <random>
#include <thread>
#include <type_traits>
#include <vector>

namespace {

// ---- binary16 with a rounding after every operation -------------------------
struct Half {
  _Float16 v;
  Half() : v(0) {}
  explicit Half(float f) : v(static_cast<_Float16>(f)) {}
  explicit Half(double d) : v(static_cast<_Float16>(d)) {}
  float f() const { return static_cast<float>(v); }
};

template <typename T>
struct Limits {
  static T max() { return std::numeric_limits<T>::max(); }
  static T min() { return std::numeric_limits<T>::min(); }
  static T zero() { return T(0); }
  static T one() { return T(1); }
};
template <>
struct Limits<Half> {
  static Half max() { return Half(65504.0f); }
  static Half min() { return Half(6.103515625e-05f); }
  static Half zero() { return Half(0.0f); }
  static Half one() { return Half(1.0f); }
};

template <typename T> inline T add(T a, T b) { return static_cast<T>(a + b); }
template <typename T> inline T mul(T a, T b) { return static_cast<T>(a * b); }
template <typename T> inline bool lt(T a, T b) { return a < b; }
template <typename T> inline bool nz(T a) { return a != T(0); }
template <> inline Half add(Half a, Half b) { return Half(a.f() + b.f()); }
template <> inline Half mul(Half a, Half b) { return Half(a.f() * b.f()); }
template <> inline bool lt(Half a, Half b) { return a.f() < b.f(); }
template <> inline bool nz(Half a) { return a.f() != 0.0f; }

// ---- the five functors (Operators.h:20-100) ---------------------------------
enum Op { kMultiply = 0, kAdd = 1, kMin = 2, kMax = 3, kAnd = 4 };

template <typename T, int OP>
struct Functor;
template <typename T>
struct Functor<T, kAdd> {
  static T Apply(T a, T b) { return add(a, b); }
  static T identity() { return Limits<T>::zero(); }
};
template <typename T>
struct Functor<T, kMultiply> {
  static T Apply(T a, T b) { return mul(a, b); }
  static T identity() { return Limits<T>::one(); }
};
template <typename T>
struct Functor<T, kAnd> {
  static T Apply(T a, T b) { return (nz(a) && nz(b)) ? Limits<T>::one() : Limits<T>::zero(); }
  static T identity() { return Limits<T>::one(); }
};
template <typename T>
struct Functor<T, kMin> {
  static T Apply(T a, T b) { return lt(a, b) ? a : b; }
  static T identity() { return Limits<T>::max(); }
};
template <typename T>
struct Functor<T, kMax> {
  static T Apply(T a, T b) { return lt(b, a) ? a : b; }
  static T identity() { return Limits<T>::min(); }
};

// ---- Naive (Utility.h:18-42), restricted to a row range ---------------------
template <typename T, int MAP, int RED>
void NaiveRows(const T *a, const T *b, T *c, long size_n, long size_k,
               long size_m, bool transposed_a, long row_begin, long row_end) {
  using Map = Functor<T, MAP>;
  using Red = Functor<T, RED>;
  for (long n = row_begin; n < row_end; ++n) {
    for (long m = 0; m < size_m; ++m) {
      T acc = Red::identity();
      for (long k = 0; k < size_k; ++k) {
        const T elem_a = transposed_a ? a[k * size_n + n] : a[n * size_k + k];
        const T elem_b = b[k * size_m + m];
        acc = Red::Apply(acc, Map::Apply(elem_a, elem_b));
      }
      c[n * size_m + m] = acc;
    }
  }
}

template <typename T, int MAP, int RED>
void NaiveThreaded(const T *a, const T *b, T *c, long n, long k, long m,
                   bool ta, long row_begin, long row_end, int threads) {
  if (threads <= 1 || row_end - row_begin < 2) {
    NaiveRows<T, MAP, RED>(a, b, c, n, k, m, ta, row_begin, row_end);
    return;
  }
  std::vector<std::thread> pool;
  const long rows = row_end - row_begin;
  const long per = (rows + threads - 1) / threads;
  for (int t = 0; t < threads; ++t) {
    const long lo = row_begin + t * per;
    const long hi = std::min(row_end, lo + per);
    if (lo >= hi) break;
    pool.emplace_back(NaiveRows<T, MAP, RED>, a, b, c, n, k, m, ta, lo, hi);
  }
  for (auto &t : pool) t.join();
}

template <typename T, int MAP>
int DispatchReduce(int red, const T *a, const T *b, T *c, long n, long k,
                   long m, bool ta, long r0, long r1, int threads) {
  switch (red) {
    case kMultiply: NaiveThreaded<T, MAP, kMultiply>(a, b, c, n, k, m, ta, r0, r1, threads); return 0;
    case kAdd: NaiveThreaded<T, MAP, kAdd>(a, b, c, n, k, m, ta, r0, r1, threads); return 0;
    case kMin: NaiveThreaded<T, MAP, kMin>(a, b, c, n, k, m, ta, r0, r1, threads); return 0;
    case kMax: NaiveThreaded<T, MAP, kMax>(a, b, c, n, k, m, ta, r0, r1, threads); return 0;
    case kAnd: NaiveThreaded<T, MAP, kAnd>(a, b, c, n, k, m, ta, r0, r1, threads); return 0;
  }
  return 2;
}

template <typename T>
int DispatchMap(int map, int red, const void *a, const void *b, void *c, long n,
                long k, long m, bool ta, long r0, long r1, int threads) {
  const T *pa = static_cast<const T *>(a);
  const T *pb = static_cast<const T *>(b);
  T *pc = static_cast<T *>(c);
  switch (map) {
    case kMultiply: return DispatchReduce<T, kMultiply>(red, pa, pb, pc, n, k, m, ta, r0, r1, threads);
    case kAdd: return DispatchReduce<T, kAdd>(red, pa, pb, pc, n, k, m, ta, r0, r1, threads);
    case kMin: return DispatchReduce<T, kMin>(red, pa, pb, pc, n, k, m, ta, r0, r1, threads);
    case kMax: return DispatchReduce<T, kMax>(red, pa, pb, pc, n, k, m, ta, r0, r1, threads);
    case kAnd: return DispatchReduce<T, kAnd>(red, pa, pb, pc, n, k, m, ta, r0, r1, threads);
  }
  return 2;
}

// ---- input recipe (TestSimulation.cpp:46-55) --------------------------------
template <typename T>
struct Caster {
  static T from_real(double d) { return static_cast<T>(d); }
  static T from_int(unsigned long u) { return static_cast<T>(u); }
};
template <>
struct Caster<Half> {
  static Half from_real(double d) { return Half(d); }
  static Half from_int(unsigned long u) { return Half(static_cast<double>(u)); }
};

template <typename T, bool INTEGRAL>
void Fill(T *a, size_t na, T *b, size_t nb, unsigned seed) {
  std::default_random_engine rng(seed);
  if (INTEGRAL) {
    std::uniform_int_distribution<unsigned long> dist(1, 10);
    for (size_t i = 0; i < na; ++i) a[i] = Caster<T>::from_int(dist(rng));
    for (size_t i = 0; i < nb; ++i) b[i] = Caster<T>::from_int(dist(rng));
  } else {
    std::uniform_real_distribution<double> dist(1, 10);
    for (size_t i = 0; i < na; ++i) a[i] = Caster<T>::from_real(dist(rng));
    for (size_t i = 0; i < nb; ++i) b[i] = Caster<T>::from_real(dist(rng));
  }
}

// ---- acceptance criterion (TestSimulation.cpp:75-92) ------------------------
template <typename T>
long VerifyFloat(const T *test, const T *ref, size_t count) {
  for (size_t i = 0; i < count; ++i) {
    const T diff = std::abs(test[i] - ref[i]);
    if (diff / ref[i] > static_cast<T>(1e-3)) return static_cast<long>(i);
  }
  return -1;
}
long VerifyHalf(const Half *test, const Half *ref, size_t count) {
  // `half` is not std::is_floating_point, so the reference takes the exact
  // branch for it (TestSimulation.cpp:81-85).
  for (size_t i = 0; i < count; ++i) {
    if (test[i].f() != ref[i].f()) return static_cast<long>(i);
  }
  return -1;
}
template <typename T>
long VerifyInt(const T *test, const T *ref, size_t count) {
  for (size_t i = 0; i < count; ++i) {
    if (test[i] != ref[i]) return static_cast<long>(i);
  }
  return -1;
}

}  // namespace

// dtype codes match include/mm_b200.h (MM_DTYPE_*).
enum { kHalf = 0, kFloat = 1, kDouble = 2, kInt32 = 3, kUint32 = 4, kUint8 = 5 };

extern "C" {

int oracle_dtype_size(int dtype) {
  switch (dtype) {
    case kHalf: return 2;
    case kFloat: return 4;
    case kDouble: return 8;
    case kInt32: return 4;
    case kUint32: return 4;
    case kUint8: return 1;
  }
  return 0;
}

// Rows [row_begin, row_end) of C = A (x) B; `threads` row-parallel workers
// (1 == exactly the reference's single-threaded loop nest).
int oracle_naive_rows(int dtype, int map_op, int reduce_op, int transposed_a,
                      const void *a, const void *b, void *c, long n, long k,
                      long m, long row_begin, long row_end, int threads) {
  const bool ta = transposed_a != 0;
  if (row_begin < 0 || row_end > n || row_begin > row_end) return 3;
  switch (dtype) {
    case kHalf: return DispatchMap<Half>(map_op, reduce_op, a, b, c, n, k, m, ta, row_begin, row_end, threads);
    case kFloat: return DispatchMap<float>(map_op, reduce_op, a, b, c, n, k, m, ta, row_begin, row_end, threads);
    case kDouble: return DispatchMap<double>(map_op, reduce_op, a, b, c, n, k, m, ta, row_begin, row_end, threads);
    case kInt32: return DispatchMap<int>(map_op, reduce_op, a, b, c, n, k, m, ta, row_begin, row_end, threads);
    case kUint32: return DispatchMap<unsigned>(map_op, reduce_op, a, b, c, n, k, m, ta, row_begin, row_end, threads);
    case kUint8: return DispatchMap<unsigned char>(map_op, reduce_op, a, b, c, n, k, m, ta, row_begin, row_end, threads);
  }
  return 1;
}

int oracle_naive(int dtype, int map_op, int reduce_op, int transposed_a,
                 const void *a, const void *b, void *c, long n, long k, long m,
                 int threads) {
  return oracle_naive_rows(dtype, map_op, reduce_op, transposed_a, a, b, c, n, k,
                           m, 0, n, threads);
}

int oracle_fill(int dtype, void *a, size_t na, void *b, size_t nb, unsigned seed) {
  switch (dtype) {
    case kHalf: Fill<Half, false>(static_cast<Half *>(a), na, static_cast<Half *>(b), nb, seed); return 0;
    case kFloat: Fill<float, false>(static_cast<float *>(a), na, static_cast<float *>(b), nb, seed); return 0;
    case kDouble: Fill<double, false>(static_cast<double *>(a), na, static_cast<double *>(b), nb, seed); return 0;
    case kInt32: Fill<int, true>(static_cast<int *>(a), na, static_cast<int *>(b), nb, seed); return 0;
    case kUint32: Fill<unsigned, true>(static_cast<unsigned *>(a), na, static_cast<unsigned *>(b), nb, seed); return 0;
    case kUint8: Fill<unsigned char, true>(static_cast<unsigned char *>(a), na, static_cast<unsigned char *>(b), nb, seed); return 0;
  }
  return 1;
}

// Returns the flat index of the first mismatch under the reference's
// criterion, -1 if none, -2 on a bad dtype.
long oracle_verify(int dtype, const void *test, const void *ref, size_t count) {
  switch (dtype) {
    case kHalf: return VerifyHalf(static_cast<const Half *>(test), static_cast<const Half *>(ref), count);
    case kFloat: return VerifyFloat(static_cast<const float *>(test), static_cast<const float *>(ref), count);
    case kDouble: return VerifyFloat(static_cast<const double *>(test), static_cast<const double *>(ref), count);
    case kInt32: return VerifyInt(static_cast<const int *>(test), static_cast<const int *>(ref), count);
    case kUint32: return VerifyInt(static_cast<const unsigned *>(test), static_cast<const unsigned *>(ref), count);
    case kUint8: return VerifyInt(static_cast<const unsigned char *>(test), static_cast<const unsigned char *>(ref), count);
  }
  return -2;
}

}  // extern "C"
