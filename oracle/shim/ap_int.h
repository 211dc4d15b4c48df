// TEST INFRASTRUCTURE ONLY — never linked into the product library.
//
// Minimal stand-in for the Xilinx Vitis-HLS header <ap_int.h>, which the
// reference includes (hlslib/include/hlslib/xilinx/DataPack.h:8-9,
// kernel/Compute.cpp:161-165) but which is not vendored in the reference checkout and
// does not exist in this image.  It lets the reference's own, unmodified
// sources (kernel/{Compute,Memory,Top}.cpp, test/TestSimulation.cpp,
// include/Utility.h) compile IN PLACE with plain g++ so that oracle/_ref holds
// the real reference behaviour to pin the oracle restatement against.
//
// Only the subset of the ap_(u)int API those files touch is provided:
//   * tightly packed little-endian storage (sizeof(ap_uint<512>) == 64), since
//     DataPack reinterprets the bytes (DataPack.h:31-37) and the kernel indexes
//     MemoryPack_t[] directly over the host vectors;
//   * construction from / conversion to integers, ++ with wrap to W bits;
//   * range(hi, lo) read/write proxies.
#pragma once

#include <cstddef>
#include <cstdint>
#include <cstring>
#include <iostream>   // Vitis' ap_int.h pulls these in transitively; DataPack.h:163-168 relies on it
#include <sstream>
#include <stdexcept>
#include <string>

template <int W>
struct ap_uint;

namespace ap_shim {

// Read `nbits` bits starting at bit `lo` of a little-endian byte array.
inline void copy_bits(unsigned char *dst, int dst_lo, const unsigned char *src,
                      int src_lo, int nbits) {
  if ((dst_lo % 8 == 0) && (src_lo % 8 == 0) && (nbits % 8 == 0)) {
    std::memcpy(dst + dst_lo / 8, src + src_lo / 8, nbits / 8);
    return;
  }
  for (int i = 0; i < nbits; ++i) {
    const int s = src_lo + i, d = dst_lo + i;
    const unsigned bit = (src[s / 8] >> (s % 8)) & 1u;
    dst[d / 8] = static_cast<unsigned char>((dst[d / 8] & ~(1u << (d % 8))) |
                                            (bit << (d % 8)));
  }
}

template <int W>
struct RangeRef {
  ap_uint<W> &ref;
  int hi, lo;
  template <int K>
  operator ap_uint<K>() const;
  template <int K>
  RangeRef &operator=(ap_uint<K> const &rhs);
};

template <int W>
struct ConstRangeRef {
  ap_uint<W> const &ref;
  int hi, lo;
  template <int K>
  operator ap_uint<K>() const;
};

}  // namespace ap_shim

template <int W>
struct ap_uint {
  static_assert(W > 0, "width must be positive");
  static constexpr int kBytes = (W + 7) / 8;
  unsigned char b[kBytes];

  ap_uint() { std::memset(b, 0, kBytes); }
  ap_uint(unsigned long long v) { assign(v); }
  ap_uint(long long v) { assign(static_cast<unsigned long long>(v)); }
  ap_uint(unsigned long v) { assign(v); }
  ap_uint(long v) { assign(static_cast<unsigned long long>(v)); }
  ap_uint(unsigned v) { assign(v); }
  ap_uint(int v) { assign(static_cast<unsigned long long>(v)); }

  void assign(unsigned long long v) {
    std::memset(b, 0, kBytes);
    for (int i = 0; i < kBytes && i < 8; ++i) {
      b[i] = static_cast<unsigned char>(v >> (8 * i));
    }
    mask();
  }

  void mask() {
    if (W % 8 != 0) {
      b[kBytes - 1] &= static_cast<unsigned char>((1u << (W % 8)) - 1u);
    }
  }

  unsigned long long to_u64() const {
    unsigned long long v = 0;
    for (int i = 0; i < kBytes && i < 8; ++i) {
      v |= static_cast<unsigned long long>(b[i]) << (8 * i);
    }
    return v;
  }

  operator unsigned long long() const { return to_u64(); }

  ap_uint &operator++() {
    assign(to_u64() + 1);
    return *this;
  }
  ap_uint operator++(int) {
    ap_uint old = *this;
    ++(*this);
    return old;
  }

  ap_shim::RangeRef<W> range(int hi, int lo) {
    return ap_shim::RangeRef<W>{*this, hi, lo};
  }
  ap_shim::ConstRangeRef<W> range(int hi, int lo) const {
    return ap_shim::ConstRangeRef<W>{*this, hi, lo};
  }
  ap_shim::RangeRef<W> range() { return range(W - 1, 0); }
  ap_shim::ConstRangeRef<W> range() const { return range(W - 1, 0); }
};

template <int W>
struct ap_int : public ap_uint<W> {
  using ap_uint<W>::ap_uint;
};

namespace ap_shim {

template <int W>
template <int K>
RangeRef<W>::operator ap_uint<K>() const {
  ap_uint<K> out;
  const int n = hi - lo + 1;
  copy_bits(out.b, 0, ref.b, lo, n < K ? n : K);
  return out;
}

template <int W>
template <int K>
RangeRef<W> &RangeRef<W>::operator=(ap_uint<K> const &rhs) {
  const int n = hi - lo + 1;
  copy_bits(ref.b, lo, rhs.b, 0, n < K ? n : K);
  return *this;
}

template <int W>
template <int K>
ConstRangeRef<W>::operator ap_uint<K>() const {
  ap_uint<K> out;
  const int n = hi - lo + 1;
  copy_bits(out.b, 0, ref.b, lo, n < K ? n : K);
  return out;
}

}  // namespace ap_shim

// Vitis' ap_int.h transitively provides `half` (hls_half.h); the reference
// names the type unconditionally in include/Utility.h:125-129.
#include "hls_half.h"
