// Run-time (dtype, map, reduce, flags) -> compile-time (T, Map, Reduce) for the four families of CUDA-core semiring
// kernels: the product, the accumulate call, the witness call and the closure.  Every family takes the same kernels'
// operators, so C of the accumulate, witness and closure calls is what the product computes.
#include "common.cuh"
#include "semiring_kernel.cuh"

namespace mm {

namespace {

template <template <typename, class, class> class Family, typename T>
int by_map(int map_op, int reduce_op, const GemmArgs &g, unsigned *w) {
  switch (map_op) {
    case MM_OP_MULTIPLY: return launch_semiring_for<Family, T, MM_OP_MULTIPLY>(reduce_op, g, w);
    case MM_OP_ADD: return launch_semiring_for<Family, T, MM_OP_ADD>(reduce_op, g, w);
    case MM_OP_MIN: return launch_semiring_for<Family, T, MM_OP_MIN>(reduce_op, g, w);
    case MM_OP_MAX: return launch_semiring_for<Family, T, MM_OP_MAX>(reduce_op, g, w);
    case MM_OP_AND: return launch_semiring_for<Family, T, MM_OP_AND>(reduce_op, g, w);
  }
  if constexpr (std::is_same<T, float>::value) {  // the hardware min/max variants (internal operator codes)
    switch (map_op) {
      case MM_OP_MIN_FAST: return launch_semiring_for<Family, float, MM_OP_MIN_FAST>(reduce_op, g, w);
      case MM_OP_MAX_FAST: return launch_semiring_for<Family, float, MM_OP_MAX_FAST>(reduce_op, g, w);
    }
  }
  return -1;
}

template <template <typename, class, class> class Family>
int launch(int dtype, int map_op, int reduce_op, const GemmArgs &g, unsigned *w, const char *what) {
  int rc = -1;
  switch (dtype) {
    case MM_DTYPE_HALF: rc = by_map<Family, __half>(map_op, reduce_op, g, w); break;
    case MM_DTYPE_FLOAT: {
      // Min / Max on float use FMNMX unless the caller asked for the literal C++ semantics
      auto fast = [&](int op) {
        if (g.flags & MM_FLAG_EXACT) return op;
        return op == MM_OP_MIN ? int(MM_OP_MIN_FAST) : (op == MM_OP_MAX ? int(MM_OP_MAX_FAST) : op);
      };
      rc = by_map<Family, float>(fast(map_op), fast(reduce_op), g, w);
      break;
    }
    case MM_DTYPE_DOUBLE: rc = by_map<Family, double>(map_op, reduce_op, g, w); break;
    case MM_DTYPE_INT32: rc = by_map<Family, int>(map_op, reduce_op, g, w); break;
    case MM_DTYPE_UINT32: rc = by_map<Family, unsigned>(map_op, reduce_op, g, w); break;
    case MM_DTYPE_UINT8: rc = by_map<Family, unsigned char>(map_op, reduce_op, g, w); break;
    case MM_DTYPE_BFLOAT16: rc = by_map<Family, __nv_bfloat16>(map_op, reduce_op, g, w); break;
    default: return fail(MM_ERR_INVALID, "unknown data type");
  }
  if (rc < 0) return fail(MM_ERR_INVALID, std::string("unknown map operator, or a reduce with no ") + what + " kernel");
  if (rc != 0) {
    return fail(MM_ERR_CUDA, std::string(what) + " kernel launch: " + cudaGetErrorString(static_cast<cudaError_t>(rc)));
  }
  return MM_OK;
}

}  // namespace

int launch_semiring(int dtype, int map_op, int reduce_op, const GemmArgs &g) {
  return launch<SemiringProduct>(dtype, map_op, reduce_op, g, nullptr, "semiring");
}

int launch_semiring_accumulate(int dtype, int map_op, int reduce_op, const GemmArgs &g) {
  return launch<SemiringAccumulate>(dtype, map_op, reduce_op, g, nullptr, "accumulate");
}

int launch_semiring_witness(int dtype, int map_op, int reduce_op, const GemmArgs &g, unsigned *w) {
  return launch<SemiringWitness>(dtype, map_op, reduce_op, g, w, "witness");
}

int launch_semiring_closure(int dtype, int map_op, int reduce_op, int flags, void *d, unsigned n, unsigned batch,
                            cudaStream_t stream) {
  GemmArgs g{d, d, d, n, n, n, flags, stream};
  g.batch.count = batch;
  return launch<SemiringClosure>(dtype, map_op, reduce_op, g, nullptr, "closure");
}

}  // namespace mm
