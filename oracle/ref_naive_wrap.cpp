// TEST INFRASTRUCTURE ONLY.  Compiled by oracle/build.py once per
// (MM_DATA_TYPE, MM_MAP_OP, MM_REDUCE_OP[, MM_TRANSPOSED_A]) against the
// REFERENCE'S OWN headers where they lie in the reference checkout (with the vendor
// headers the reference does not ship replaced by oracle/shim/), into
// oracle/_ref/libref_naive_<cfg>.so.  The function body that runs is the
// reference's Naive<> template, include/Utility.h:18-42, instantiated with the
// reference's hlslib::op functors (hlslib/include/hlslib/xilinx/Operators.h).
#include "Utility.h"

extern "C" {

void ref_naive(const void *a, const void *b, void *c, int n, int k, int m) {
  Naive<OperatorMap, OperatorReduce>(static_cast<Data_t const *>(a),
                                     static_cast<Data_t const *>(b),
                                     static_cast<Data_t *>(c), n, k, m);
}

// ReferenceImplementation (Utility.h:105-111): with no BLAS in this image it is
// CallBLAS' fallback (Utility.h:66-74) -> Naive<>, after a warning on stdout.
void ref_reference_implementation(const void *a, const void *b, void *c,
                                  unsigned n, unsigned k, unsigned m) {
  ReferenceImplementation(static_cast<Data_t const *>(a),
                          static_cast<Data_t const *>(b),
                          static_cast<Data_t *>(c), n, k, m);
}

int ref_sizeof_data_t() { return static_cast<int>(sizeof(Data_t)); }
int ref_seed() { return kSeed; }
int ref_memory_width_k() { return kMemoryWidthK; }
int ref_memory_width_m() { return kMemoryWidthM; }

}  // extern "C"
