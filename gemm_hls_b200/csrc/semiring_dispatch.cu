// Run-time (dtype, map, reduce) -> compile-time instantiation of the semiring tile kernels, plain and accumulate.
#include "common.cuh"
#include "semiring_kernel.cuh"

namespace mm {

namespace {

// ACC: the accumulate kernels (semiring_accumulate_inst.cu), otherwise the plain ones (semiring_inst.cu)
template <typename T, int MAP_OP, bool ACC>
int launch_for(int reduce_op, const GemmArgs &g, bool ta, bool ring) {
  if constexpr (ACC) {
    return launch_semiring_accumulate_for<T, MAP_OP>(reduce_op, g.a, g.b, g.c, g.n, g.k, g.m, ta, ring, g.batch, g.stream);
  } else {
    return launch_semiring_for<T, MAP_OP>(reduce_op, g.a, g.b, g.c, g.n, g.k, g.m, ta, ring, g.batch, g.stream);
  }
}

template <typename T, bool ACC>
int by_map(int map_op, int reduce_op, const GemmArgs &g, bool ta, bool ring) {
  switch (map_op) {
    case MM_OP_MULTIPLY: return launch_for<T, MM_OP_MULTIPLY, ACC>(reduce_op, g, ta, ring);
    case MM_OP_ADD: return launch_for<T, MM_OP_ADD, ACC>(reduce_op, g, ta, ring);
    case MM_OP_MIN: return launch_for<T, MM_OP_MIN, ACC>(reduce_op, g, ta, ring);
    case MM_OP_MAX: return launch_for<T, MM_OP_MAX, ACC>(reduce_op, g, ta, ring);
    case MM_OP_AND: return launch_for<T, MM_OP_AND, ACC>(reduce_op, g, ta, ring);
  }
  return -1;
}

// float only: the hardware min/max variants (internal operator codes)
template <bool ACC>
int by_map_float(int map_op, int reduce_op, const GemmArgs &g, bool ta, bool ring) {
  switch (map_op) {
    case MM_OP_MIN_FAST: return launch_for<float, MM_OP_MIN_FAST, ACC>(reduce_op, g, ta, ring);
    case MM_OP_MAX_FAST: return launch_for<float, MM_OP_MAX_FAST, ACC>(reduce_op, g, ta, ring);
  }
  return by_map<float, ACC>(map_op, reduce_op, g, ta, ring);
}

template <bool ACC>
int launch(int dtype, int map_op, int reduce_op, const GemmArgs &g_in) {
  GemmArgs g = g_in;
  if (g.dry_run) g.a = nullptr;  // launch_semiring_typed: null A = load the kernel, launch nothing
  const bool ta = (g.flags & MM_FLAG_TRANSPOSED_A) != 0;
  const bool ring = g.tuning ? g.tuning->semiring_ring() : true;
  int rc = -1;
  switch (dtype) {
    case MM_DTYPE_HALF: rc = by_map<__half, ACC>(map_op, reduce_op, g, ta, ring); break;
    case MM_DTYPE_FLOAT: {
      // Min / Max on float use FMNMX unless the caller asked for the literal C++ semantics
      auto fast = [&](int op) {
        if (g.flags & MM_FLAG_EXACT) return op;
        return op == MM_OP_MIN ? int(MM_OP_MIN_FAST) : (op == MM_OP_MAX ? int(MM_OP_MAX_FAST) : op);
      };
      rc = by_map_float<ACC>(fast(map_op), fast(reduce_op), g, ta, ring);
      break;
    }
    case MM_DTYPE_DOUBLE: rc = by_map<double, ACC>(map_op, reduce_op, g, ta, ring); break;
    case MM_DTYPE_INT32: rc = by_map<int, ACC>(map_op, reduce_op, g, ta, ring); break;
    case MM_DTYPE_UINT32: rc = by_map<unsigned, ACC>(map_op, reduce_op, g, ta, ring); break;
    case MM_DTYPE_UINT8: rc = by_map<unsigned char, ACC>(map_op, reduce_op, g, ta, ring); break;
    case MM_DTYPE_BFLOAT16: rc = by_map<__nv_bfloat16, ACC>(map_op, reduce_op, g, ta, ring); break;
    default: return fail(MM_ERR_INVALID, "unknown data type");
  }
  if (rc < 0) return fail(MM_ERR_INVALID, "unknown map/reduce operator");
  if (rc != 0) return fail(MM_ERR_CUDA, std::string("semiring kernel launch: ") + cudaGetErrorString(static_cast<cudaError_t>(rc)));
  return MM_OK;
}

}  // namespace

int launch_semiring(int dtype, int map_op, int reduce_op, const GemmArgs &g) {
  return launch<false>(dtype, map_op, reduce_op, g);
}

// C <- Reduce(C_old, product): the same kernel choice (FMNMX for float Min / Max without MM_FLAG_EXACT, the ring
// kernel for row-major 4-byte types unless MM_TUNE_SEMIRING_RING = 0), with the accumulate kernels.
int launch_semiring_accumulate(int dtype, int map_op, int reduce_op, const GemmArgs &g) {
  return launch<true>(dtype, map_op, reduce_op, g);
}

}  // namespace mm
